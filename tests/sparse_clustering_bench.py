"""Timings of PartialMiniBatchKMeans and SpectralClustering on sparse CSR blocks on an H100 (not a test).

    python tests/sparse_clustering_bench.py [--reps 10] [--small] [--out file.json]

Workloads (those of tests/kmeans_sparse_bench.py): hashed 4M x 2^20 (Zipf columns, 60 draws a row, fp32 values) and
one-hot 10M x 1024 (8 groups of 128 categories), fp32 values.  Passes are timed with CUDA events, median of --reps after
a warm-up, alternated in the same process with a torch composition of the same result, and the outputs compared:
  colsum / embed (l = 100 keep rows, k = 8)  bkm_csr_kernel_colsum_chunk / bkm_csr_nystrom_embed_chunk  vs
      bkm_csr_assign_chunk mode 2 into an (n, l) float64 buffer, then torch exp / sum / @ W
  SpectralClustering.fit (n_components = 100, n_clusters = 8)
  one mini-batch step on a 1M-row block at k = 100, split into the assign pass, the block's transpose, the label sums,
      the step kernel and the host read
  PartialMiniBatchKMeans.fit over the 1M-row blocks  vs  scikit-learn's MiniBatchKMeans.partial_fit on the same host
      blocks (scipy CSR)
"""
import argparse
import json
import os
import sys
import time
import warnings

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from glm_sparse_bench import card, hashed, onehot, timed  # noqa: E402


def _wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def bench_nystrom(res, be, blk, d, reps, l=100, k=8, gamma=0.5):
    from dask_ml_b200._sparse import _SparseData

    crow, col, val, n = blk
    X = _SparseData([blk], d, be)
    keep = np.sort(np.random.RandomState(2).choice(n, l, replace=False))
    from dask_ml_b200.cluster.k_means import _dense_centres

    C = _dense_centres(X.global_rows(keep), d, be)
    pack = be.sparse_pack_centers(C)
    W = torch.randn((l, k), dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    c = torch.empty(l, dtype=torch.float64, device="cuda")
    e = torch.empty((n, k), dtype=torch.float32, device="cuda")
    buf = torch.empty((n, l), dtype=torch.float64, device="cuda")
    ref = {}

    def ours_colsum():
        be.csr_kernel_colsum(blk, d, pack, l, gamma, c, first=True)

    def torch_colsum():
        be.csr_assign_chunk(blk, d, pack, l, out=buf, mode=2)
        ref["c"] = torch.exp(buf * -gamma).sum(0)

    def ours_embed():
        be.csr_nystrom_embed(blk, d, pack, l, gamma, W, e)

    def torch_embed():
        be.csr_assign_chunk(blk, d, pack, l, out=buf, mode=2)
        K = torch.exp((buf - buf.min(1, keepdim=True)[0]) * -gamma)
        v = K @ W
        ref["e"] = (v / v.norm(dim=1, keepdim=True)).to(torch.float32)

    res["colsum_ms"], res["colsum_torch_ms"] = timed([ours_colsum, torch_colsum], reps)
    res["embed_ms"], res["embed_torch_ms"] = timed([ours_embed, torch_embed], reps)
    ours_colsum(), torch_colsum(), ours_embed(), torch_embed()
    torch.cuda.synchronize()
    res["colsum_max_rel_diff"] = float(((c - ref["c"]).abs() / ref["c"].abs()).max().item())
    res["embed_max_abs_diff"] = float((e - ref["e"]).abs().max().item())
    del buf, ref
    torch.cuda.empty_cache()


def bench_minibatch_step(res, be, blk, d, reps, k=100):
    from dask_ml_b200.cluster.minibatch import _SparseMiniBatchState
    from dask_ml_b200._sparse import _SparseData

    crow, col, val, n = blk
    m = min(n, 1_000_000)
    e1 = int(crow[m].item())
    b1 = (crow[: m + 1], col[:e1], val[:e1], m)
    X = _SparseData([b1], d, be)
    seeds = np.sort(np.random.RandomState(1).choice(m, k, replace=False))
    C0 = X.global_rows(seeds).toarray().astype(np.float64)
    st = _SparseMiniBatchState(be, C0, np.zeros(k))
    lab = torch.empty(m, dtype=torch.int32, device="cuda")
    pack = st.packs[st.cur]
    keep = {}

    def assign():
        be.csr_assign_chunk(b1, d, pack, k, labels=lab, counts=st.counts, dist_sum=st.inertia, first=True)

    def transpose():
        keep["csc"] = be.csr_transpose_chunk(b1, d)

    transpose()

    def label_sums():
        be.csc_label_sums_chunk(keep["csc"], d, lab, k, st.sums, first=True)

    pin, pout = st.packs[0], st.packs[1]
    w_in, w_out = st.Wb[0], st.Wb[1]

    def step():
        be.sparse_minibatch_step(st.red, pin, w_in, pout, w_out, k, d)

    def host_read():
        st.start_read()
        st.finish_read()

    def whole():
        st.step(be, [b1])
        st.start_read()
        st.finish_read()

    t = timed([assign, transpose, label_sums, step, host_read, whole], reps)
    for name, v in zip(("step_assign_ms", "step_transpose_ms", "step_label_sums_ms", "step_kernel_ms",
                        "step_host_read_ms", "step_whole_ms"), t):
        res[name] = v
    res["step_rows"], res["step_k"] = m, k
    del keep
    torch.cuda.empty_cache()


def bench_fits(res, blk, d, small):
    import scipy.sparse as sp
    from sklearn.cluster import MiniBatchKMeans

    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import PartialMiniBatchKMeans, SpectralClustering

    crow, col, val, n = blk
    rows = 1_000_000 if not small else 10_000
    parts = []
    for r0 in range(0, n, rows):
        r1 = min(n, r0 + rows)
        e0, e1 = int(crow[r0].item()), int(crow[r1].item())
        parts.append(torch.sparse_csr_tensor(crow[r0:r1 + 1] - e0, col[e0:e1], val[e0:e1], size=(r1 - r0, d)))
    Xc = ChunkedArray(parts)
    res["spectral_fit_s"], _ = _wall(lambda: SpectralClustering(n_clusters=8, n_components=100, gamma=0.5,
                                                                random_state=0).fit(Xc))
    np.random.seed(0)
    res["minibatch_fit_s"], est = _wall(lambda: PartialMiniBatchKMeans(n_clusters=100, random_state=0).fit(Xc))
    np.random.seed(0)
    order = list(range(len(parts)))
    np.random.shuffle(order)
    host = [sp.csr_matrix((p.values().cpu().numpy(), p.col_indices().cpu().numpy(), p.crow_indices().cpu().numpy()),
                          shape=tuple(p.shape)) for p in parts]
    sk = MiniBatchKMeans(n_clusters=100, random_state=0, n_init=1)
    t0 = time.perf_counter()
    for i in order:
        sk.partial_fit(host[i])
    res["sklearn_partial_fit_s"] = time.perf_counter() - t0
    res["minibatch_vs_sklearn_centre_max_abs_diff"] = float(np.abs(est.cluster_centers_ - sk.cluster_centers_).max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--small", action="store_true", help="tiny sizes (a check of the script, not a measurement)")
    a = ap.parse_args()
    warnings.simplefilter("ignore")
    from dask_ml_b200.engine import CudaBackend

    be = CudaBackend()
    results = {"card": card()}
    gen = torch.Generator(device="cuda").manual_seed(0)
    n1, n2 = (4_000_000, 10_000_000) if not a.small else (40_000, 100_000)
    for name in ("hashed", "onehot"):
        if name == "hashed":
            d = 1 << 20
            crow, col, val = hashed(n1, d, 60, gen)
            n = n1
        else:
            d = 1024
            crow, col, val = onehot(n2, 8, 128, gen)
            n = n2
        blk = (crow, col, val, n)
        res = {"n": n, "p": d, "nnz": int(col.numel())}
        bench_nystrom(res, be, blk, d, a.reps)
        bench_minibatch_step(res, be, blk, d, a.reps)
        bench_fits(res, blk, d, a.small)
        print(name, json.dumps(res), flush=True)
        results[name] = res
        del crow, col, val, blk
        torch.cuda.empty_cache()
    results["card_after"] = card()
    print(json.dumps(results, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
