"""Timing of the sparse passes of the linear models on one H100 (not part of the suite).

Two workloads, one CSR block each, float32 values:
  hashed   4M rows x 2^20 features, ~60 Zipf-distributed entries per row (text-like)
  onehot   10M rows x 1024 features: 8 columns x 128 categories, one category in 50 % of the rows

Per block it times, with CUDA events after a warm-up, each pass alternated in the same process with a torch
composition of the same result: the transpose build (against torch's CSR -> CSC conversion), the gradient evaluation
(row pass + column pass, against torch.sparse.mm for X beta and X^T r through torch's CSC), the predict pass (against
torch.sparse.mm), and for the one-hot block the Newton evaluation, whose Gram is compared with the dense
bkm_gram_weighted_chunk on a densified slice that fits.  Outputs are compared at the timed sizes.  Each time is set
against its HBM floor: the bytes of CSR, CSC and r / w read once over 3.35 TB/s.  Then one whole
LogisticRegression(solver="lbfgs").fit per workload.  The card's name, power limit and clock are read in the same run.

    python tests/glm_sparse_bench.py [--reps 10] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                                       text=True).strip().splitlines()[-1]
    except Exception as e:                                 # pragma: no cover
        return "unknown (%s)" % e


def timed(fns, reps):
    """Median ms of each fn, the fns alternated rep by rep (after one warm-up call each)."""
    for f in fns:
        f()
    torch.cuda.synchronize()
    times = [[] for _ in fns]
    for _ in range(reps):
        for k, f in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            torch.cuda.synchronize()
            times[k].append(a.elapsed_time(b))
    return [float(np.median(t)) for t in times]


def hashed(n, d, per_row, gen):
    """Zipf columns (p(rank k) ~ 1 / k), hashed to random places, duplicates within a row removed."""
    u = torch.rand((n, per_row), generator=gen, device="cuda", dtype=torch.float64)
    rank = torch.floor(torch.exp(u * np.log(d))).to(torch.int64) - 1          # log-uniform: density ~ 1 / k
    perm = torch.randperm(d, generator=gen, device="cuda")
    cols, _ = torch.sort(perm[rank.clamp_(0, d - 1)], dim=1)
    keep = torch.ones_like(cols, dtype=torch.bool)
    keep[:, 1:] = cols[:, 1:] != cols[:, :-1]
    crow = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    crow[1:] = torch.cumsum(keep.sum(1), 0)
    col = cols[keep]
    val = torch.rand(col.numel(), generator=gen, device="cuda", dtype=torch.float32) + 0.5
    return crow, col, val


def onehot(n, groups, cats, gen):
    hot = torch.rand((n, groups), generator=gen, device="cuda") < 0.5
    other = torch.randint(1, cats, (n, groups), generator=gen, device="cuda")
    cat = torch.where(hot, torch.zeros_like(other), other)
    col = (cat + torch.arange(groups, device="cuda") * cats).reshape(-1)
    crow = torch.arange(0, n * groups + 1, groups, dtype=torch.int64, device="cuda")
    return crow, col, torch.ones(col.numel(), dtype=torch.float32, device="cuda")


def bench_block(name, crow, col, val, n, d, reps, newton):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.engine import CudaBackend
    from dask_ml_b200.linear_model import LogisticRegression

    be = CudaBackend()
    nnz = int(col.numel())
    blk = (crow, col, val, n)
    gen = torch.Generator(device="cuda").manual_seed(1)
    bstar = torch.randn(d + 1, generator=gen, device="cuda", dtype=torch.float64) / np.sqrt(nnz / n)
    X64 = torch.sparse_csr_tensor(crow, col, val.double(), size=(n, d))
    eta = (torch.sparse.mm(X64, bstar[:d, None])[:, 0] + bstar[d])
    y = (torch.rand(n, generator=gen, device="cuda", dtype=torch.float64) < torch.sigmoid(eta)).double()
    beta = bstar * 0.5
    res = {"workload": name, "n": n, "d": d, "nnz": nnz}

    # the transpose, once per fit, against torch's conversion
    out = {}

    def ours_t():
        out["csc"] = be.csr_transpose_chunk(blk, d)

    def torch_t():
        out["tcsc"] = X64.to_sparse_csc()

    t_ours, t_torch = timed([ours_t, torch_t], max(2, reps // 3))
    csc = out["csc"]
    tc = out["tcsc"]
    assert int(csc[3][0].item()) == 0
    assert torch.equal(csc[0], tc.ccol_indices()) and torch.equal(csc[1].long(), tc.row_indices())
    assert torch.equal(csc[2].double(), tc.values())
    n_slots = int(csc[3][2].item())
    csr_b = 8 * (n + 1) + 12 * nnz
    csc_b = 8 * (d + 1) + 8 * nnz
    res["transpose_ms"] = t_ours
    res["transpose_torch_ms"] = t_torch
    res["transpose_floor_ms"] = (csr_b + csc_b) / HBM * 1e3

    # gradient evaluation: row pass + column pass
    XT = torch.sparse_csr_tensor(tc.ccol_indices(), tc.row_indices(), tc.values(), size=(d, n))
    red = torch.empty(d + 2, dtype=torch.float64, device="cuda")
    r = torch.empty(n, dtype=torch.float64, device="cuda")
    tg = {}

    def ours_g():
        be.glm_csr_pass_chunk(blk, d, y, beta, 0, 0, r=r, grad=red, first=True)
        be.csc_matvec_chunk(csc, d, r, red, first=True)

    def torch_g():
        e = torch.sparse.mm(X64, beta[:d, None])[:, 0] + beta[d]
        rr = torch.sigmoid(e) - y
        tg["g"] = torch.sparse.mm(XT, rr[:, None])[:, 0]

    g_ours, g_torch = timed([ours_g, torch_g], reps)
    scale = float(torch.sparse.mm(torch.sparse_csr_tensor(XT.crow_indices(), XT.col_indices(), XT.values().abs(),
                                                          size=(d, n)), r.abs()[:, None]).max())
    res["grad_max_abs_diff_over_scale"] = float((red[:d] - tg["g"]).abs().max()) / max(scale, 1e-300)
    res["grad_ms"] = g_ours
    res["grad_torch_ms"] = g_torch
    res["grad_floor_ms"] = (csr_b + csc_b + 8 * n * 3) / HBM * 1e3

    # predict pass
    mu = torch.empty(n, dtype=torch.float64, device="cuda")
    tp = {}

    def ours_p():
        be.glm_csr_pass_chunk(blk, d, None, beta, 0, 2, out=mu)

    def torch_p():
        tp["mu"] = torch.sigmoid(torch.sparse.mm(X64, beta[:d, None])[:, 0] + beta[d])

    p_ours, p_torch = timed([ours_p, torch_p], reps)
    res["predict_max_abs_diff"] = float((mu - tp["mu"]).abs().max())
    res["predict_ms"] = p_ours
    res["predict_torch_ms"] = p_torch
    res["predict_floor_ms"] = (csr_b + 8 * n) / HBM * 1e3

    if newton:
        w = torch.empty(n, dtype=torch.float64, device="cuda")
        hrow = torch.empty(d + 1, dtype=torch.float64, device="cuda")
        G = torch.empty((d, d), dtype=torch.float64, device="cuda")

        def ours_n():
            be.glm_csr_pass_chunk(blk, d, y, beta, 0, 1, r=r, w=w, grad=red, hrow=hrow, first=True)
            be.csc_matvec_chunk(csc, d, r, red, v2=w, out2=hrow, first=True)
            be.gram_weighted_csr_chunk(blk, csc, d, w, G, n_slots, first=True)

        # the dense Gram on a densified slice that fits, against the sparse Gram of the same slice
        m = min(n, 1 << 20)
        sl = (crow[: m + 1], col[: int(crow[m])], val[: int(crow[m])], m)
        dense = torch.sparse_csr_tensor(sl[0], sl[1], sl[2], size=(m, d)).to_dense()
        wm = torch.rand(m, generator=gen, device="cuda", dtype=torch.float64) * 0.25
        csc_m = be.csr_transpose_chunk(sl, d)
        slots_m = int(csc_m[3][2].item())
        Gs = torch.empty((d, d), dtype=torch.float64, device="cuda")
        Gd = torch.empty((d, d), dtype=torch.float64, device="cuda")

        def ours_gs():
            be.gram_weighted_csr_chunk(sl, csc_m, d, wm, Gs, slots_m, first=True)

        def dense_gs():
            be.gram_weighted_chunk(dense, wm, Gd, first=True)

        n_ours, = timed([ours_n], reps)
        gs_ours, gs_dense = timed([ours_gs, dense_gs], reps)
        res["gram_slice_rows"] = m
        res["gram_slice_rel_diff"] = float((Gs - Gd).abs().max() / Gd.abs().max())
        res["gram_slice_ms"] = gs_ours
        res["gram_slice_dense_ms"] = gs_dense
        res["newton_ms"] = n_ours
        res["newton_floor_ms"] = (2 * csr_b + csc_b + 8 * n * 5) / HBM * 1e3
        del dense

    # one whole fit
    Xc = ChunkedArray([torch.sparse_csr_tensor(crow, col, val, size=(n, d))])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    est = LogisticRegression(solver="lbfgs").fit(Xc, ChunkedArray([y]))
    torch.cuda.synchronize()
    res["fit_lbfgs_s"] = time.perf_counter() - t0
    res["fit_coef_finite"] = bool(np.isfinite(est.coef_).all())
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--small", action="store_true", help="tiny sizes (a check of the script, not a measurement)")
    a = ap.parse_args()
    info = card()
    gen = torch.Generator(device="cuda").manual_seed(0)
    n1, n2 = (4_000_000, 10_000_000) if not a.small else (40_000, 100_000)
    results = {"card": info}
    crow, col, val = hashed(n1, 1 << 20, 60, gen)
    results["hashed"] = bench_block("hashed", crow, col, val, n1, 1 << 20, a.reps, newton=False)
    del crow, col, val
    torch.cuda.empty_cache()
    crow, col, val = onehot(n2, 8, 128, gen)
    results["onehot"] = bench_block("onehot", crow, col, val, n2, 1024, a.reps, newton=True)
    results["card_after"] = card()
    print(json.dumps(results, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
