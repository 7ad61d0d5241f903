"""Speed of GaussianNB's passes on one GPU (run on an H100: python tests/nb_bench.py [--out FILE]).

Shapes: 10M x 64 fp32 with K = 10 and K = 256, and 8M x 128 bf16 with K = 10.  Per pass, CUDA-event times of the
kernels (bkm_class_moments_chunk mode 0 and mode 1, bkm_nb_jll_chunk with the arg-max epilogue and with the
log-probability epilogue) alternated in the same process with the torch composition they replace: ``index_add_`` sums
and counts of the float64 rows, and a broadcasted ``((x - theta)^2 w).sum(-1)`` per block of 2^28 / (K d) rows followed by
``argmax`` or ``log_softmax``.  Outputs are checked against each other.  Reports achieved GB/s (the bytes of X and y
read plus the output written) against the 3.35 TB/s floor computed from the shapes, with the card's name and power
limit from the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dask_ml_b200.engine import CudaBackend  # noqa: E402

PEAK_BW = 3.35e12
BLOCK = 1 << 18


def _time(fn, reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        ev[0].record()
        fn()
        ev[1].record()
        torch.cuda.synchronize()
        ts.append(ev[0].elapsed_time(ev[1]))
    return float(np.median(ts))


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = torch.cuda.get_device_name()
    return q


def _pair(name, fused, torched, reps, byts, err, meta):
    tf, tt = [], []
    for _ in range(3):                             # alternate the two in the same process
        tf.append(_time(fused, reps))
        tt.append(_time(torched, reps))
    t_f, t_t = min(tf), min(tt)
    return dict(meta, pass_=name, fused_ms=t_f, torch_ms=t_t, gbps=byts / t_f / 1e6, floor_ms=byts / PEAK_BW * 1e3,
                err=err)


def run(n, d, K, dt, reps):
    be = CudaBackend()
    g = torch.Generator(device="cuda").manual_seed(0)
    y = torch.randint(0, K, (n,), device="cuda", generator=g)
    means = torch.randn((K, d), device="cuda", generator=g, dtype=torch.float64) * 2
    X = (means[y] + torch.randn((n, d), device="cuda", generator=g, dtype=torch.float64)).to(dt)
    cls = y.to(torch.int32)
    esz = X.element_size()
    meta = dict(n=n, d=d, K=K, dtype=str(dt))
    res = []
    S = torch.empty((K, d), dtype=torch.float64, device="cuda")
    C = torch.empty((K,), dtype=torch.float64, device="cuda")

    def fused_sums():
        be.class_moments_chunk(X, cls, K, S, C, first=True)

    def torch_sums():
        s = torch.zeros((K, d), dtype=torch.float64, device="cuda")
        c = torch.zeros((K,), dtype=torch.float64, device="cuda")
        for i in range(0, n, BLOCK * 4):
            s.index_add_(0, y[i:i + BLOCK * 4], X[i:i + BLOCK * 4].double())
        c.index_add_(0, y, torch.ones(n, dtype=torch.float64, device="cuda"))
        return s, c

    fused_sums()
    s_ref, c_ref = torch_sums()
    err = float((S - s_ref).abs().max() / s_ref.abs().max())
    assert torch.equal(C, c_ref)
    res.append(_pair("moments pass 1", fused_sums, torch_sums, reps, n * d * esz + n * 4, err, meta))
    theta = (S / C[:, None]).contiguous()
    Q = torch.empty((K, d), dtype=torch.float64, device="cuda")

    def fused_sq():
        be.class_moments_chunk(X, cls, K, Q, theta=theta, first=True)

    def torch_sq():
        q = torch.zeros((K, d), dtype=torch.float64, device="cuda")
        for i in range(0, n, BLOCK * 4):
            q.index_add_(0, y[i:i + BLOCK * 4], (X[i:i + BLOCK * 4].double() - theta[y[i:i + BLOCK * 4]]) ** 2)
        return q

    fused_sq()
    q_ref = torch_sq()
    err = float((Q - q_ref).abs().max() / q_ref.abs().max())
    res.append(_pair("moments pass 2", fused_sq, torch_sq, reps, n * d * esz + n * 4, err, meta))

    sigma = Q / C[:, None]
    w = (1.0 / sigma).contiguous()
    logc = (torch.log(C / n) - 0.5 * torch.log(2 * np.pi * sigma).sum(1)).contiguous()
    lab = torch.empty((n,), dtype=torch.int32, device="cuda")
    out = torch.empty((n, K), dtype=torch.float64, device="cuda")
    tf_ = theta.float()
    wf = w.float()

    jb = max(1024, (1 << 28) // (K * d))              # rows per block of the broadcasted (rows, K, d) product

    def torch_jll(i):
        x = X[i:i + jb].float() if dt != torch.float64 else X[i:i + jb]
        t, ww = (tf_, wf) if dt != torch.float64 else (theta, w)
        s = (((x[:, None, :] - t[None]) ** 2) * ww[None]).sum(-1)
        return logc[None] - 0.5 * s.double()

    def fused_lab():
        be.nb_jll_chunk(X, theta, w, logc, labels=lab)

    def torch_lab():
        return torch.cat([torch_jll(i).argmax(1) for i in range(0, n, jb)])

    fused_lab()
    lr = torch_lab()
    err = float((lab.long() != lr).float().mean())
    res.append(_pair("predict labels", fused_lab, torch_lab, reps, n * d * esz + n * 4, err, meta))

    def fused_lp():
        be.nb_jll_chunk(X, theta, w, logc, out=out)

    def torch_lp():
        for i in range(0, n, jb):
            out_t[i:i + jb] = torch.log_softmax(torch_jll(i), 1)

    out_t = torch.empty_like(out)
    fused_lp()
    torch_lp()
    err = max(float((out[i:i + BLOCK] - out_t[i:i + BLOCK]).abs().max()) for i in range(0, n, BLOCK))
    res.append(_pair("predict log-proba", fused_lp, torch_lp, max(2, reps // 2), n * d * esz + n * K * 8, err, meta))
    del X, out, out_t
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the row counts (rehearsal)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rows = []
    for n, d, K, dt in ((10_000_000, 64, 10, torch.float32), (10_000_000, 64, 256, torch.float32),
                        (8_000_000, 128, 10, torch.bfloat16)):
        rows += run(max(1, int(n * a.scale)), d, K, dt, a.reps)
        _show(rows[-4:])
    card = _card()
    print("card:", card)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(card=card, rows=rows), f, indent=1)


def _show(rows):
    for r in rows:
        print("%-18s %9d x %3d K=%3d %-14s fused %8.3f ms  torch %8.3f ms  %6.0f GB/s  floor %6.3f ms  err %.1e"
              % (r["pass_"], r["n"], r["d"], r["K"], r["dtype"], r["fused_ms"], r["torch_ms"], r["gbps"],
                 r["floor_ms"], r["err"]), flush=True)


if __name__ == "__main__":
    main()
