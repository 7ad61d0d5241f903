"""SimpleImputer's passes against their torch compositions, timed with CUDA events and alternated in one process:

    statistics (mean)       impute.missing_stats                 vs  torch.nanmean in float64
    median                  impute.median_statistics             vs  torch.nanmedian(dim=0)
    most_frequent           impute.mode_statistics               vs  per column torch.unique(col[mask], counts), arg-max
    transform               SimpleImputer.transform              vs  torch.where(isnan, stats, X) and cat of the mask

Shapes: 10M x 64 fp32 with 10 % NaN, 8M x 128 bf16, 10M x 64 fp64.  The mode pass runs on categorical columns (16
distinct values: contention on few table slots) and on continuous ones (all distinct: the largest tables), its two
extremes.  Besides each whole pass, the kernels are timed on their own: the statistics kernel over every block, and
for the first column group of the mode pass the table reset, the counting over every block and the best-entry
reduction (with the number of groups, which each repeat all three).  Each line reports the median time and the HBM
floor of the pass: the bytes it must move over 3.35 TB/s (the H100 SXM data sheet), one JSON line per measurement.

    python tests/impute_bench.py [--rows-scale 1.0] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def torch_mode(X, mask):
    out = []
    for j in range(X.shape[1]):
        u, c = torch.unique(X[:, j][~mask[:, j]], return_counts=True)
        out.append(u[torch.argmax(c)])
    return torch.stack(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows-scale", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "impute_bench needs a GPU"
    from dask_ml_b200.engine import DeviceData
    from dask_ml_b200.cluster import k_means as km
    from dask_ml_b200 import _keytables, impute

    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                               text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        power = "unknown"
    be = km._get_backend()
    g = torch.Generator(device="cuda").manual_seed(0)
    for n, d, dt in ((10_000_000, 64, torch.float32), (8_000_000, 128, torch.bfloat16), (10_000_000, 64, torch.float64)):
        n = int(n * args.rows_scale)
        X = torch.randn((n, d), device="cuda", generator=g, dtype=torch.float32).to(dt)
        X[torch.rand((n, d), device="cuda", generator=g) < 0.1] = float("nan")
        esz = X.element_size()
        data = DeviceData([X[i:i + (1 << 21)] for i in range(0, n, 1 << 21)], be)
        mask = torch.isnan(X)
        rec = {"gpu": name, "power_limit": power, "shape": [n, d], "dtype": str(dt).replace("torch.", "")}

        def report(pass_, ours, theirs, floor_bytes):
            r = dict(rec, **{"pass": pass_, "ms": round(ours, 3), "torch_ms": round(theirs, 3),
                             "hbm_floor_ms": round(floor_bytes / HBM * 1e3, 3),
                             "x_floor": round(ours / (floor_bytes / HBM * 1e3), 2)})
            print(json.dumps(r), flush=True)

        report("mean", timed(lambda: impute.missing_stats(data, True, float("nan")), args.reps),
               timed(lambda: torch.nanmean(X.double(), dim=0), args.reps), n * d * esz)
        acc = torch.zeros((4, d), dtype=torch.float64, device="cuda")
        shift = torch.zeros(d, dtype=torch.float64, device="cuda")

        def stats_kernel():
            for i, x in enumerate(data.chunks):
                be.impute_stats_chunk(x, True, float("nan"), shift, acc, first=i == 0)

        report("stats_kernel", timed(stats_kernel, args.reps), timed(lambda: torch.nanmean(X.double(), dim=0),
                                                                       args.reps), n * d * esz)
        rounds = {torch.float32: 4, torch.bfloat16: 2, torch.float64: 8}[dt]
        report("median", timed(lambda: impute.median_statistics(data, True, float("nan")), args.reps),
               timed(lambda: torch.nanmedian(X, dim=0), args.reps), rounds * n * d * esz)
        valid = (n - mask.sum(0)).cpu().numpy().astype(np.float64)
        for kind in ("categorical", "continuous"):
            if kind == "categorical":
                Y = torch.randint(0, 16, (n, d), device="cuda", generator=g).to(dt)
                Y[mask] = float("nan")
            else:
                Y = X
            yd = DeviceData([Y[i:i + (1 << 21)] for i in range(0, n, 1 << 21)], be)
            cost = [16 * _keytables.capacity(m, dt) for m in valid]
            gw, used = 1, cost[0]
            while gw < d and used + cost[gw] <= impute.MODE_BUDGET:
                used += cost[gw]
                gw += 1
            caps = cost[:gw]
            off_h = np.concatenate([[0], np.cumsum([c // 16 for c in caps])]).astype(np.int64)
            total = int(off_h[-1])
            keys = torch.empty(total, dtype=torch.int64, device="cuda")
            counts = torch.empty(total, dtype=torch.int64, device="cuda")
            off = torch.as_tensor(off_h, device="cuda")
            first_x = yd.chunks[0][:0, :gw]
            t_reset = timed(lambda: be.mode_count_chunk(first_x, True, float("nan"), keys, counts, off, total,
                                                        first=True), args.reps)

            def count():
                be.mode_count_chunk(first_x, True, float("nan"), keys, counts, off, total, first=True)
                for x in yd.chunks:
                    be.mode_count_chunk(x[:, :gw], True, float("nan"), keys, counts, off, total)

            t_count = timed(count, args.reps) - t_reset
            t_best = timed(lambda: be.mode_best(keys, counts, off, gw, total), args.reps)
            groups = -(-d // gw)
            print(json.dumps(dict(rec, **{"pass": "most_frequent_%s_group" % kind, "group_columns": gw,
                                          "groups": groups, "table_bytes": 16 * total, "reset_ms": round(t_reset, 3),
                                          "count_ms": round(t_count, 3), "best_ms": round(t_best, 3),
                                          "count_hbm_floor_ms": round(n * 32 * -(-gw * esz // 32) / HBM * 1e3, 3)})),
                  flush=True)
            del keys, counts
            report("most_frequent_" + kind,
                   timed(lambda: impute.mode_statistics(yd, True, float("nan"), valid, valid), args.reps),
                   timed(lambda: torch_mode(Y, mask), 1), n * d * esz)
            del Y, yd
        est = impute.SimpleImputer(strategy="mean", add_indicator=True).fit(data)
        st = torch.as_tensor(est.statistics_, device="cuda").to(dt)
        report("transform", timed(lambda: est.transform(data), args.reps),
               timed(lambda: torch.cat([torch.where(mask, st, X), mask.to(dt)], dim=1), args.reps),
               n * d * esz * 3)
        del X, data, mask
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
