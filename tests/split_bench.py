"""Speed of the split and the scoring passes on one GPU (run on an H100: python tests/split_bench.py [--out FILE]).

Shapes: 10M x 64 fp32 and 8M x 128 bf16, each with an int64 y, in blocks of 2M rows.  CUDA-event times, every pass
alternated in the same process with the torch composition it replaces, and the outputs compared:
  * indices (bkm_split_indices_chunk, one block) against ``torch.randperm``; once, numpy's
    ``RandomState(seed).permutation`` on the host, the serial shuffle the permutation replaces;
  * the gather of X and of y (bkm_gather_rows_chunk) against ``X[idx]``: GB/s over ``count * (8 + 2 * row_bytes)``
    bytes (the index, the row read and the row written) against the HBM floor (3.35 TB/s);
  * the whole ``train_test_split(X, y)`` against ``randperm`` + ``X[idx]`` / ``y[idx]`` per block and part;
  * each metric mode on 10M rows against its torch composition.
The card's name and power limit come from the same run.  Fails without a GPU.
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
from dask_ml_b200 import ChunkedArray  # noqa: E402
from dask_ml_b200 import _lib  # noqa: E402
from dask_ml_b200.engine import CudaBackend  # noqa: E402
from dask_ml_b200.model_selection import train_test_split  # noqa: E402
from nb_bench import _card, _pair  # noqa: E402

BLOCK = 2_000_000


def run_split(n, d, dt, reps):
    be = CudaBackend()
    g = torch.Generator(device="cuda").manual_seed(0)
    Xb = [torch.randn((min(BLOCK, n - s), d), generator=g, device="cuda", dtype=torch.float32).to(dt)
          for s in range(0, n, BLOCK)]
    yb = [torch.randint(0, 2, (b.shape[0],), generator=g, device="cuda") for b in Xb]
    X, y = ChunkedArray(Xb), ChunkedArray(yb)
    meta = dict(n=n, d=d, dtype=str(dt), block=BLOCK)
    x0, y0, c = Xb[0], yb[0], Xb[0].shape[0]
    row_bytes = d * x0.element_size()
    idx = be.split_indices_chunk(1, c, 0, c, 0)
    assert torch.equal(idx.sort().values, torch.arange(c, device="cuda"))
    res, keep = [], {}

    def f_idx():
        keep["i"] = be.split_indices_chunk(1, c, 0, c, 0)

    def t_idx():
        keep["ti"] = torch.randperm(c, device="cuda")

    def f_gx():
        keep["gx"] = be.gather_rows_chunk(x0, idx)

    def t_gx():
        keep["tgx"] = x0[idx]

    def f_gy():
        keep["gy"] = be.gather_rows_chunk(y0, idx)

    def t_gy():
        keep["tgy"] = y0[idx]

    def f_all():
        keep["all"] = train_test_split(X, y, test_size=0.2, random_state=0)

    def t_all():
        out = []
        for xb, yy in zip(Xb, yb):
            p = torch.randperm(xb.shape[0], device="cuda")
            k = xb.shape[0] // 5
            out.append((xb[p[k:]], xb[p[:k]], yy[p[k:]], yy[p[:k]]))
        keep["tall"] = out

    for f in (f_idx, t_idx, f_gx, t_gx, f_gy, t_gy, f_all, t_all):
        f()
    torch.cuda.synchronize()
    ok_x, ok_y = bool(torch.equal(keep["gx"], keep["tgx"])), bool(torch.equal(keep["gy"], keep["tgy"]))
    res.append(_pair("indices (one block)", f_idx, t_idx, reps, c * 8, dict(bijection=True), meta))
    res.append(_pair("gather X (one block)", f_gx, t_gx, reps, c * (8 + 2 * row_bytes), dict(equal=ok_x), meta))
    res.append(_pair("gather y (one block)", f_gy, t_gy, reps, c * (8 + 2 * 8), dict(equal=ok_y), meta))
    keep.clear()
    res.append(_pair("train_test_split(X, y)", f_all, t_all, max(2, reps // 4), n * (8 + 2 * row_bytes + 16),
                     dict(), meta))
    keep.clear()
    t0 = time.perf_counter()
    np.random.RandomState(1).permutation(c)
    res.append(dict(meta, pass_="numpy RandomState.permutation (one block, host)", host_ms=(time.perf_counter() - t0) * 1e3))
    return res


def run_metrics(n, reps):
    be = CudaBackend()
    g = torch.Generator(device="cuda").manual_seed(1)
    meta = dict(n=n)
    t = torch.randn(n, generator=g, device="cuda", dtype=torch.float64) + 10
    p = t + torch.randn(n, generator=g, device="cuda", dtype=torch.float64)
    yi = torch.randint(0, 2, (n,), generator=g, device="cuda")
    yp = torch.where(torch.rand(n, generator=g, device="cuda") < 0.8, yi, 1 - yi)
    pr = torch.rand(n, generator=g, device="cuda", dtype=torch.float64)
    cls = yi.to(torch.int32)
    shift = t[:1].clone()
    acc4 = torch.empty((4, 1), dtype=torch.float64, device="cuda")
    acc2 = torch.empty(2, dtype=torch.float64, device="cuda")
    keep = {}

    def f_err():
        be.metric_chunk(t, p, _lib.METRIC_ERR, acc4, shift=shift, first=True)

    def t_err():
        dl = p - t
        keep["err"] = torch.stack([(dl * dl).sum(), dl.abs().sum(), (t - shift).sum(), ((t - shift) ** 2).sum()])

    def f_eq():
        be.metric_chunk(yi, yp, _lib.METRIC_EQ, acc2, first=True)

    def t_eq():
        keep["eq"] = (yi == yp).sum(dtype=torch.float64)

    def f_ll():
        be.metric_chunk(cls, pr, _lib.METRIC_LOGLOSS, acc2, eps=1e-15, first=True)

    def t_ll():
        q = pr.clamp(1e-15, 1 - 1e-15)
        keep["ll"] = -torch.where(yi == 1, q, 1 - q).log().sum()

    res = []
    for name, f, tf, byts, acc, key, pick in (("ERR (mse, mae, r2 sums)", f_err, t_err, 16 * n, acc4, "err", None),
                                              ("EQ (accuracy)", f_eq, t_eq, 16 * n, acc2, "eq", 0),
                                              ("LOGLOSS", f_ll, t_ll, 12 * n, acc2, "ll", 0)):
        f(); tf()
        torch.cuda.synchronize()
        got = acc.reshape(-1) if pick is None else acc.reshape(-1)[pick]
        err = float(((got - keep[key]).abs() / keep[key].abs().clamp_min(1e-300)).max())
        res.append(_pair(name, f, tf, reps, byts, dict(rel=err), meta))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--scale", type=float, default=1.0, help="shrink the shapes (rehearsals)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("split_bench.py needs a CUDA device")
    card = _card()
    rows = []
    for n, d, dt in ((10_000_000, 64, torch.float32), (8_000_000, 128, torch.bfloat16)):
        rows += run_split(int(n * a.scale), d, dt, a.reps)
        torch.cuda.empty_cache()
    rows += run_metrics(int(10_000_000 * a.scale), a.reps)
    for r in rows:
        r["card"] = card
        print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
