"""Manual probe (not collected by pytest): how wrong can the tensor path be WITHOUT the float64 re-check?
Runs the tensor-core kernel with BKM_FLAG_NO_RECHECK and reports, over the rows whose label differs from the float64
arg-min, the largest float64 margin relative to ||x||^2 + max||c||^2 — the quantity the near-tie bound tau
(bkm_api.cu: tau_for) must dominate.  Run on a GPU:  python tests/tau_probe.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from dask_ml_b200.engine import CudaBackend
from dask_ml_b200 import _lib

be = CudaBackend(flags=_lib.FLAG_FORCE_TC | _lib.FLAG_NO_RECHECK)
worst_all = 0.0
for (n, d, k, kind) in [(4_000_000, 64, 256, "blobs"), (4_000_000, 64, 256, "uniform"), (2_000_000, 41, 100, "blobs"),
                        (2_000_000, 16, 64, "uniform"), (2_000_000, 64, 256, "scaled")]:
    g = torch.Generator(device=be.device).manual_seed(n + d + k)
    if kind == "uniform":
        X = torch.rand((n, d), device=be.device, generator=g) * 20 - 10
    else:
        cent = torch.empty((k // 2, d), device=be.device).uniform_(-10, 10, generator=g)
        X = cent[torch.randint(0, k // 2, (n,), device=be.device, generator=g)] + torch.randn((n, d), device=be.device, generator=g)
        if kind == "scaled":
            X = X * torch.logspace(-3, 3, d, device=be.device)
    X = be.to_device(X, torch.float32)
    C = X[torch.randperm(n, device=be.device, generator=g)[:k]].double().contiguous()
    pack = be.pack_centers(C, torch.float32)
    labels = be.empty((n,), torch.int32)
    be.assign_chunk(X, pack, k, labels, None, True, None)
    torch.cuda.synchronize()
    cn = (C * C).sum(1)
    worst = 0.0; nbad = 0
    for s in range(0, n, 1 << 18):
        xb = X[s:s + (1 << 18)].double()
        d2 = (xb * xb).sum(1, keepdim=True) + cn[None, :] - 2.0 * xb @ C.T
        best = d2.min(1)
        got = d2.gather(1, labels[s:s + xb.shape[0]].long()[:, None])[:, 0]
        bad = got > best.values
        if bool(bad.any()):
            rel = (got[bad] - best.values[bad]) / ((xb[bad] ** 2).sum(1) + cn.max())
            worst = max(worst, float(rel.max())); nbad += int(bad.sum())
    tau = (8.0 * (3.0 * ((d + 7) // 8)) ** 0.5 + 16.0) * 2.0 ** -24
    print("%-8s n=%d d=%d k=%d: %d labels differ from float64 without the re-check; worst relative margin %.3e; tau %.3e (headroom %.1fx)"
          % (kind, n, d, k, nbad, worst, tau, tau / worst if worst else float("inf")))
    worst_all = max(worst_all, worst)
print("worst over all:", worst_all)
