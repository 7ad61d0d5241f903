"""Speed of the two PCA passes on one GPU (run on an H100: python tests/pca_bench.py [--out FILE]).

Shapes: 10M x 64 fp32 and 8M x 128 bf16.  Per pass, CUDA-event times of the fused kernels (bkm_gram_chunk,
bkm_project_chunk with k = 16 and k = 64) alternated in the same process with the torch composition
Xc = X.double() - mu; Xc.T @ Xc and Xc @ W.T, whose outputs are checked against the kernels'.  Reports achieved GB/s
(the bytes of X read plus the output written) and fp64 TFLOP/s against 3.35 TB/s and 67 TFLOP/s, naming the bound, with
the card's name and power limit.  The Gram kernel computes only the 64x64 tiles on or above the diagonal: its TFLOP/s and
floor count the products it issues (2 n 64^2 per computed tile); "effective" is 2 n d^2 over the same time.  The
projection issues 2 n d k (no padding at these shapes).
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

PEAK_BW, PEAK_F64 = 3.35e12, 67e12


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


def run(n, d, dt, reps):
    be = CudaBackend()
    g = torch.Generator(device="cuda").manual_seed(0)
    X = (torch.randn((n, d), device="cuda", generator=g) * 2 + 5).to(dt)
    mu = X[: 1 << 16].double().mean(0)
    G = torch.empty((d, d), dtype=torch.float64, device="cuda")
    m = torch.empty((d,), dtype=torch.float64, device="cuda")
    esz = X.element_size()
    res = []

    def fused_gram():
        be.gram_chunk(X, mu, m, G, first=True)

    def torch_gram():
        Xc = X.double() - mu
        return Xc.T @ Xc

    ref = torch_gram()
    fused_gram()
    err = float((G - ref).abs().max() / ref.abs().max())
    tf, tt = [], []
    for _ in range(3):                         # alternate the two in the same process
        tf.append(_time(fused_gram, reps))
        tt.append(_time(torch_gram, reps))
    t_f, t_t = min(tf), min(tt)
    nb = (d + 63) // 64
    flops, byts = 2.0 * n * 64 * 64 * (nb * (nb + 1) // 2), float(n * d * esz)
    bound = "fp64 tensor" if flops / PEAK_F64 > byts / PEAK_BW else "HBM"
    res.append(dict(pass_="gram", n=n, d=d, dtype=str(dt), fused_ms=t_f, torch_ms=t_t, rel_err=err,
                    gbps=byts / t_f / 1e6, tflops=flops / t_f / 1e9, tflops_effective=2.0 * n * d * d / t_f / 1e9,
                    floor_ms=max(flops / PEAK_F64, byts / PEAK_BW) * 1e3, bound=bound))
    for k in (16, 64):
        W = torch.randn((k, d), dtype=torch.float64, device="cuda", generator=g)
        out = torch.empty((n, k), dtype=torch.float32, device="cuda")

        def fused_proj():
            be.project_chunk(X, mu, W, out=out)

        def torch_proj():
            return ((X.double() - mu) @ W.T).float()

        r = torch_proj()
        fused_proj()
        err = float((out - r).abs().max() / r.abs().max())
        tf, tt = [], []
        for _ in range(3):
            tf.append(_time(fused_proj, reps))
            tt.append(_time(torch_proj, reps))
        t_f, t_t = min(tf), min(tt)
        flops, byts = 2.0 * n * d * k, float(n * d * esz + n * k * 4)
        bound = "fp64 tensor" if flops / PEAK_F64 > byts / PEAK_BW else "HBM"
        res.append(dict(pass_="project k=%d" % k, n=n, d=d, dtype=str(dt), fused_ms=t_f, torch_ms=t_t, rel_err=err,
                        gbps=byts / t_f / 1e6, tflops=flops / t_f / 1e9, tflops_effective=flops / t_f / 1e9,
                        floor_ms=max(flops / PEAK_F64, byts / PEAK_BW) * 1e3, bound=bound))
    del X
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the row counts (rehearsal)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rows = [r for n, d, dt in ((10_000_000, 64, torch.float32), (8_000_000, 128, torch.bfloat16))
            for r in run(max(1, int(n * a.scale)), d, dt, a.reps)]
    card = _card()
    for r in rows:
        print("%-14s %9d x %3d %-14s fused %8.3f ms  torch %8.3f ms  %7.0f GB/s  %6.2f TFLOP/s issued (%6.2f effective)  "
              "floor %6.3f ms (%s)  "
              "rel.err %.1e" % (r["pass_"], r["n"], r["d"], r["dtype"], r["fused_ms"], r["torch_ms"], r["gbps"],
                                r["tflops"], r["tflops_effective"], r["floor_ms"], r["bound"], r["rel_err"]))
    print("card:", card)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(card=card, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
