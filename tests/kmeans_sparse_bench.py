"""Timings of the sparse KMeans passes on an H100 (not a test).

    python tests/kmeans_sparse_bench.py [--reps 10] [--small] [--out file.json]

Workloads (from tests/glm_sparse_bench.py): hashed 4M x 2^20 (Zipf columns, 60 draws a row, fp32 values), k = 100;
one-hot 10M x 1024 (8 groups of 128 categories), k = 16.  Each pass is timed with CUDA events, median of --reps after a
warm-up, alternated in the same process with a float64 torch composition of the same result, and the outputs are
compared at the timed sizes:
  assign     bkm_csr_assign_chunk (labels + counts)   vs  torch.sparse.mm(X, CT) + norms + argmin + bincount
  label sums bkm_csc_label_sums_chunk                 vs  index_add_ of the rows into a (k, p) buffer
  finalize   bkm_sparse_finalize_step                 vs  sums / counts, the shift and the norms in torch
Also: the HBM floor and the gathered bytes of the assign pass, one whole Lloyd iteration, KMeans.fit with an array init
and with k-means||, and (one-hot) the dense engine on a densified 1M-row slice against the sparse path on that slice.
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
from glm_sparse_bench import card, hashed, onehot, timed  # noqa: E402


def bench_block(name, crow, col, val, n, d, k, reps, dense_slice):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200._sparse import _SparseData
    from dask_ml_b200.cluster import KMeans
    from dask_ml_b200.cluster.k_means import _SparseLloydState
    from dask_ml_b200.engine import CudaBackend

    be = CudaBackend()
    blk = (crow, col, val, n)
    X = _SparseData([blk], d, be)
    csc = X.transposes()[0]
    nnz = int(col.numel())
    gen = torch.Generator(device="cuda").manual_seed(1)
    seeds = np.sort(np.random.RandomState(1).choice(n, k, replace=False))
    Xt = torch.sparse_csr_tensor(crow, col, val.to(torch.float64), size=(n, d))
    C = torch.from_numpy(X.global_rows(seeds).toarray().astype(np.float64)).cuda()
    C = C + 0.01 * torch.rand((k, d), generator=gen, device="cuda", dtype=torch.float64)
    pack = be.sparse_pack_centers(C)
    lab = torch.empty(n, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(k, dtype=torch.float64, device="cuda")
    sumsT = torch.empty((d, k), dtype=torch.float64, device="cuda")
    red = torch.zeros(d * k + k + 1, dtype=torch.float64, device="cuda")
    red[: d * k].view(d, k).copy_(C.t())
    red[d * k: d * k + k] = 1.0
    out_pack = torch.empty_like(pack)
    res = {"n": n, "p": d, "k": k, "nnz": nnz}

    CT = pack[: d * k].view(d, k)
    cn = pack[d * k:]
    xn = torch.zeros(n, dtype=torch.float64, device="cuda")
    rows = torch.repeat_interleave(torch.arange(n, device="cuda"), crow[1:] - crow[:-1])
    xn.index_add_(0, rows, val.to(torch.float64) ** 2)
    t_lab = [None]

    def ours_assign():
        be.csr_assign_chunk(blk, d, pack, k, labels=lab, counts=cnt, first=True)

    def torch_assign():
        d2 = xn[:, None] - 2.0 * torch.sparse.mm(Xt, CT) + cn[None, :]
        t_lab[0] = d2.argmin(1)
        torch.bincount(t_lab[0], minlength=k)

    a_ours, a_torch = timed([ours_assign, torch_assign], reps)
    ours_assign()
    torch_assign()
    torch.cuda.synchronize()
    res["assign_ms"], res["assign_torch_ms"] = a_ours, a_torch
    res["assign_labels_equal_frac"] = float((lab.long() == t_lab[0]).double().mean().item())
    res["gathered_GB"] = nnz * k * 8 / 1e9
    floor_bytes = nnz * (8 + val.element_size()) + (n + 1) * 8 + n * 4 + d * k * 8
    res["hbm_floor_ms"] = floor_bytes / 3.35e12 * 1e3

    vals64 = val.to(torch.float64)
    ref_sums = [None]

    def ours_sums():
        be.csc_label_sums_chunk(csc, d, lab, k, sumsT, first=True)

    def torch_sums():
        S = torch.zeros((k * d,), dtype=torch.float64, device="cuda")
        S.index_add_(0, lab.long()[rows] * d + col, vals64)
        ref_sums[0] = S

    s_ours, s_torch = timed([ours_sums, torch_sums], reps)
    ours_sums()
    torch_sums()
    torch.cuda.synchronize()
    res["label_sums_ms"], res["label_sums_torch_ms"] = s_ours, s_torch
    res["label_sums_max_abs_diff"] = float((sumsT.t().reshape(-1) - ref_sums[0]).abs().max().item())

    state, _ = be.loop_state_new(-1.0, 1 << 30)           # never converges: every step runs

    def ours_fin():
        be.sparse_finalize_step(red, pack, out_pack, state, k, d)

    def torch_fin():
        S = red[: d * k].view(d, k) / red[d * k: d * k + k].clamp(min=1.0)[None, :]
        ((CT - S) ** 2).sum()
        (S * S).sum(0)

    f_ours, f_torch = timed([ours_fin, torch_fin], reps)
    res["finalize_ms"], res["finalize_torch_ms"] = f_ours, f_torch

    st = _SparseLloydState(X, C.cpu().numpy())

    def one_iter():
        st.run(1, -1.0)

    res["lloyd_iteration_ms"] = timed([one_iter], max(3, reps // 2))[0]

    Xc = ChunkedArray([torch.sparse_csr_tensor(crow, col, val, size=(n, d))])
    C0 = C.cpu().numpy()
    for label, kw in (("fit_array_init_s", dict(init=C0, max_iter=10, tol=0.0)),
                      ("fit_kmeans_parallel_s", dict(init="k-means||", random_state=0, max_iter=10, tol=0.0,
                                                    init_max_iter=2))):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        est = KMeans(n_clusters=k, **kw).fit(Xc)
        torch.cuda.synchronize()
        res[label] = time.perf_counter() - t0
        res[label.replace("_s", "_n_iter")] = int(est.n_iter_)

    if dense_slice:
        m = min(n, 1_000_000)
        e = int(crow[m].item())
        Xs = torch.sparse_csr_tensor(crow[: m + 1], col[:e], val[:e], size=(m, d))
        dense = Xs.to_dense()
        C0 = C.cpu().numpy().astype(np.float32)
        for label, data in (("slice_dense_fit_s", dense), ("slice_sparse_fit_s", ChunkedArray([Xs]))):
            KMeans(n_clusters=k, init=C0, max_iter=2, tol=0.0).fit(data)       # warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            KMeans(n_clusters=k, init=C0, max_iter=10, tol=0.0).fit(data)
            torch.cuda.synchronize()
            res[label] = time.perf_counter() - t0
        del dense
    print(name, json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--small", action="store_true", help="tiny sizes (a check of the script, not a measurement)")
    a = ap.parse_args()
    results = {"card": card()}
    gen = torch.Generator(device="cuda").manual_seed(0)
    n1, n2 = (4_000_000, 10_000_000) if not a.small else (40_000, 100_000)
    crow, col, val = hashed(n1, 1 << 20, 60, gen)
    results["hashed"] = bench_block("hashed", crow, col, val, n1, 1 << 20, 100, a.reps, False)
    del crow, col, val
    torch.cuda.empty_cache()
    crow, col, val = onehot(n2, 8, 128, gen)
    results["onehot"] = bench_block("onehot", crow, col, val, n2, 1024, 16, a.reps, True)
    results["card_after"] = card()
    print(json.dumps(results, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
