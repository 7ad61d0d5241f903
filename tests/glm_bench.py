"""Speed of the linear models' passes on one GPU (run on an H100: python tests/glm_bench.py [--out FILE]).

Shapes: 10M x 64 fp32 and 8M x 128 bf16, logistic family.  CUDA-event times of one Newton iteration
(bkm_glm_pass_chunk mode 1 + bkm_gram_weighted_chunk) and of one gradient pass (mode 0), alternated in the same process
with the torch composition they replace: ``eta = X.double() @ beta``, the family terms, ``X^T r`` and, for Newton,
``(X w)^T X`` in float64.  Outputs are compared.  Reports achieved GB/s against the HBM floor (3.35 TB/s; the Newton
iteration reads X twice) and the DMMA floor of the weighted Gram at 67 TFLOP/s fp64 tensor.  As in pca_bench.py the
floor counts the products the kernel issues: it computes the 64x64 tiles on or above the diagonal in full, 2 n 64^2
flops per tile.  The card's name and power limit come from the same run.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from dask_ml_b200.engine import CudaBackend  # noqa: E402
from nb_bench import PEAK_BW, _card, _pair  # noqa: E402

PEAK_DMMA = 67e12


def run(n, d, dt, reps):
    be = CudaBackend()
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((n, d), generator=g, device="cuda", dtype=torch.float32).to(dt)
    beta = torch.randn((d + 1,), generator=g, device="cuda", dtype=torch.float64) / np.sqrt(d)
    y = (torch.rand((n,), generator=g, device="cuda", dtype=torch.float64) < 0.5).to(torch.float64)
    grad = torch.empty((d + 2,), dtype=torch.float64, device="cuda")
    hrow = torch.empty((d + 1,), dtype=torch.float64, device="cuda")
    w = torch.empty((n,), dtype=torch.float64, device="cuda")
    G = torch.empty((d, d), dtype=torch.float64, device="cuda")

    def newton():
        be.glm_pass_chunk(x, y, beta, 0, 1, grad=grad, hrow=hrow, w=w, first=True)
        be.gram_weighted_chunk(x, w, G, first=True)

    def gradient():
        be.glm_pass_chunk(x, y, beta, 0, 0, grad=grad, first=True)

    out = {}
    blk = 1 << 21

    def torch_pass(hess):
        gt = torch.zeros((d + 2,), dtype=torch.float64, device="cuda")
        Gt = torch.zeros((d, d), dtype=torch.float64, device="cuda") if hess else None
        for s in range(0, n, blk):
            xb = x[s:s + blk].double()
            eta = xb @ beta[:d] + beta[d]
            mu = torch.sigmoid(eta)
            r = mu - y[s:s + blk]
            gt[:d] += xb.T @ r
            gt[d] += r.sum()
            gt[d + 1] += (torch.nn.functional.softplus(eta) - y[s:s + blk] * eta).sum()
            if hess:
                ww = mu * (1 - mu)
                Gt += (xb * ww[:, None]).T @ xb
        out["g"], out["G"] = gt, Gt

    newton()
    torch_pass(True)
    torch.cuda.synchronize()
    eg = float(((grad - out["g"]).abs().max() / out["g"].abs().max()).item())
    eG = float(((G - out["G"]).abs().max() / out["G"].abs().max()).item())
    es = x.element_size()
    meta = dict(n=n, d=d, dtype=str(dt).replace("torch.", ""))
    xb = n * d * es
    nb = (d + 63) // 64
    nt = nb * (nb + 1) // 2                   # Gram tiles on or above the diagonal
    rows = [
        _pair("newton_iteration", newton, lambda: torch_pass(True), reps, 2 * xb + 16 * n + 8 * n,
              dict(grad=eg, gram=eG), dict(meta, dmma_floor_ms=2.0 * n * 64 * 64 * nt / PEAK_DMMA * 1e3)),
        _pair("gradient_pass", gradient, lambda: torch_pass(False), reps, xb + 8 * n, dict(grad=eg), meta),
    ]
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    card = _card()
    res = {"card": card, "rows": run(10_000_000, 64, torch.float32, args.reps) + run(8_000_000, 128, torch.bfloat16,
                                                                                      args.reps)}
    for r in res["rows"]:
        print(json.dumps(r))
    print("card:", card)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
