"""Times the encoders' passes on the GPU against their torch compositions, alternated in the same process.

    python tests/encode_bench.py [--reps 3] [--out results/encode_bench.json]

Workloads (int64 / fp32 device data, 2M-row blocks):
  A  10M x 8 int64, 16 categories per column: fit, dense float32 one-hot, CSR
  B  10M x 4 fp32, 10^4 distinct values per column: fit, CSR
  C  10M int64 labels, 1000 classes: LabelEncoder.fit_transform
  D  10M x 1 int64, ~5M distinct values: fit (the table growth path)
The torch composition: per-column torch.unique(sorted=True) for fit, torch.searchsorted for codes, zeros + scatter_ for
the dense one-hot, sparse_csr_tensor of the searchsorted indices for CSR.  Outputs are compared.  The HBM floor of each
pass is its bytes (X read once; the output written once) over 3.35 TB/s.  Prints one JSON object with the card's name
and power limit.
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
ROWS = 1 << 21


def timed(fn, reps):
    """Median of ``reps`` CUDA-event times of fn() in ms, after one warm-up call; and fn()'s last result."""
    out = fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), out


def chunked(t):
    from dask_ml_b200 import ChunkedArray

    return ChunkedArray([t[i:i + ROWS] for i in range(0, t.shape[0], ROWS)])


def torch_fit(X):
    return [torch.unique(X[:, j], sorted=True) for j in range(X.shape[1])]


def torch_codes(X, cats):
    return torch.stack([torch.searchsorted(cats[j], X[:, j].contiguous()) for j in range(X.shape[1])], 1)


def torch_dense(X, cats, dtype):
    off = np.concatenate([[0], np.cumsum([len(c) for c in cats])])
    out = torch.zeros((X.shape[0], int(off[-1])), dtype=dtype, device=X.device)
    idx = torch_codes(X, cats) + torch.as_tensor(off[:-1], device=X.device)
    out.scatter_(1, idx, 1)
    return out


def torch_csr(X, cats, dtype):
    off = np.concatenate([[0], np.cumsum([len(c) for c in cats])])
    n, d = X.shape
    idx = (torch_codes(X, cats) + torch.as_tensor(off[:-1], device=X.device)).reshape(-1)
    crow = torch.arange(0, n * d + 1, d, device=X.device)
    return torch.sparse_csr_tensor(crow, idx, torch.ones(n * d, dtype=dtype, device=X.device), size=(n, int(off[-1])))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:  # pragma: no cover
        q = "nvidia-smi failed: %s" % e
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "encode_bench.py needs a GPU"
    from dask_ml_b200.preprocessing import LabelEncoder, OneHotEncoder

    n, reps = args.n, args.reps
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"card": card(), "n": n, "reps": reps, "workloads": {}}

    def record(name, ms, floor_bytes, torch_ms=None, agree=None):
        r = {"ms": round(ms, 3), "floor_ms": round(floor_bytes / HBM * 1e3, 3), "x_floor": round(ms / (floor_bytes / HBM * 1e3), 2)}
        if torch_ms is not None:
            r["torch_ms"] = round(torch_ms, 3)
        if agree is not None:
            r["agree"] = bool(agree)
        res["workloads"][name] = r
        print(name, r, flush=True)

    # A: 10M x 8 int64, 16 categories per column
    XA = torch.randint(0, 16, (n, 8), device="cuda", generator=g) * 1000 - 7
    ca = chunked(XA)
    ms, enc = timed(lambda: OneHotEncoder(sparse=False, dtype=np.float32).fit(ca), reps)
    tms, cats = timed(lambda: torch_fit(XA), reps)
    agree = all(np.array_equal(enc.categories_[j], cats[j].cpu().numpy()) for j in range(8))
    record("A_fit_10Mx8_i64_16cat", ms, XA.numel() * 8, tms, agree)
    ms, out = timed(lambda: enc.transform(ca), reps)
    tms, want = timed(lambda: torch_dense(XA, cats, torch.float32), reps)
    agree = torch.equal(torch.cat(out.blocks), want)
    del out, want
    record("A_dense_f32", ms, XA.numel() * 8 + n * 128 * 4, tms, agree)
    enc.sparse = True
    ms, out = timed(lambda: enc.transform(ca), reps)
    tms, want = timed(lambda: torch_csr(XA, cats, torch.float32), reps)
    agree = torch.equal(torch.cat([b.col_indices() for b in out.blocks]), want.col_indices())
    del out, want
    record("A_csr_f32", ms, XA.numel() * 8 + XA.numel() * 12, tms, agree)
    del XA, ca

    # B: 10M x 4 fp32, 10^4 distinct values per column
    XB = torch.randint(0, 10000, (n, 4), device="cuda", generator=g).float() * 0.25
    cb = chunked(XB)
    ms, enc = timed(lambda: OneHotEncoder(sparse=True, dtype=np.float32).fit(cb), reps)
    tms, cats = timed(lambda: torch_fit(XB), reps)
    agree = all(np.array_equal(enc.categories_[j], cats[j].cpu().numpy()) for j in range(4))
    record("B_fit_10Mx4_f32_1e4", ms, XB.numel() * 4, tms, agree)
    ms, out = timed(lambda: enc.transform(cb), reps)
    tms, want = timed(lambda: torch_csr(XB, cats, torch.float32), reps)
    agree = torch.equal(torch.cat([b.col_indices() for b in out.blocks]), want.col_indices())
    del out, want
    record("B_csr_f32", ms, XB.numel() * 4 + XB.numel() * 12, tms, agree)
    del XB, cb

    # C: 10M int64 labels, 1000 classes
    yC = torch.randint(0, 1000, (n,), device="cuda", generator=g) * 3 + 11
    cc = chunked(yC)
    ms, out = timed(lambda: LabelEncoder().fit_transform(cc), reps)

    def torch_ft():
        u = torch.unique(yC, sorted=True)
        return torch.searchsorted(u, yC)

    tms, want = timed(torch_ft, reps)
    agree = torch.equal(torch.cat(out.blocks), want)
    record("C_label_fit_transform_10M_1000", ms, n * 8 * 2 + n * 8, tms, agree)
    del yC, cc, out, want

    # D: 10M x 1 int64, ~5M distinct: the growth path
    XD = (torch.randint(0, 5_000_000, (n, 1), device="cuda", generator=g) * 2654435761) % (1 << 40)
    cd = chunked(XD)
    ms, enc = timed(lambda: OneHotEncoder().fit(cd), reps)
    tms, cats = timed(lambda: torch_fit(XD), reps)
    agree = np.array_equal(enc.categories_[0], cats[0].cpu().numpy())
    record("D_fit_10Mx1_i64_5M", ms, XD.numel() * 8, tms, agree)
    res["distinct_D"] = int(len(enc.categories_[0]))
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
