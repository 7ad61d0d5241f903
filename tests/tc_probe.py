"""Manual probe of the tensor-core path (not collected by pytest): accuracy of the split-fp16 product and parity
with the oracle on a few shapes.  Run on a GPU:  python tests/tc_probe.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from dask_ml_b200.engine import CudaBackend
from dask_ml_b200 import _lib
from oracle import kmeans_oracle as ok

be = CudaBackend(flags=_lib.FLAG_FORCE_TC)
shapes = [(128, 64, 256), (1000, 64, 256), (40000, 64, 256), (5000, 32, 64), (3000, 16, 16),
          (7777, 40, 100), (2000, 64, 130), (300000, 64, 256)]
if len(sys.argv) > 1:
    shapes = shapes[: int(sys.argv[1])]
for (n, d, k) in shapes:
    rng = np.random.RandomState(0)
    cent = rng.uniform(-10, 10, size=(max(2, k // 2), d))
    X = (cent[rng.randint(0, len(cent), size=n)] + rng.standard_normal((n, d))).astype(np.float32)
    C = X[rng.choice(n, k, replace=n < k)].astype(np.float64) + 0.01 * rng.standard_normal((k, d))
    x = be.to_device(X, torch.float32)
    pack = be.pack_centers(torch.as_tensor(C).to(be.device), torch.float32)
    labels = be.empty((n,), torch.int32); mind2 = be.empty((n,), torch.float32)
    sums = be.zeros((k * d,), torch.float64); counts = be.zeros((k,), torch.int64); inertia = be.zeros((1,), torch.float64)
    be.lloyd_chunk(x, pack, k, labels, mind2, sums, counts, inertia)
    torch.cuda.synchronize()
    code = be.lib.bkm_debug_abort_code()
    if code:
        import ctypes
        det = (ctypes.c_uint * 64)()
        be.lib.bkm_debug_abort_detail(ctypes.cast(det, ctypes.c_void_p))
        print("ABORT first=0x%08x" % code)
        offs = [((v >> 12) & 0xfff) for v in det if v]
        base = min(offs) if offs else 0
        for w, v in enumerate(det):
            if v:
                print("  warp %2d: bar_off=%d (rel idx %+d) parity=%d cta=%d" % (w, (v >> 12) & 0xfff, (((v >> 12) & 0xfff) - base) // 8, (v >> 8) & 1, v & 0xff))
        break
    got = labels.cpu().numpy()
    (olab,), (omin,) = ok.pairwise_distances_argmin_min([X], C, metric_kwargs={"squared": True})
    bad = np.nonzero(got != olab)[0]
    X64 = X.astype(np.float64)
    if len(bad):
        gb = np.clip(got[bad], 0, k - 1)
        dg = ((X64[bad] - C[gb]) ** 2).sum(1); dw = ((X64[bad] - C[olab[bad]]) ** 2).sum(1)
        scale = (X64[bad] ** 2).sum(1) + (C ** 2).sum(1).max()
        worst = (np.abs(dg - dw) / scale).max()
    else:
        worst = 0.0
    gc = np.clip(got, 0, k - 1)
    osums = ok.centers_dense(X, gc, k)
    serr = np.abs(sums.cpu().numpy().reshape(k, d) - osums).max() / max(1e-30, np.abs(osums).max())
    cerr = np.abs(counts.cpu().numpy() - np.bincount(gc, minlength=k)).max()
    gmin = mind2.cpu().numpy().astype(np.float64)
    dsel = ((X64 - C[gc]) ** 2).sum(1)
    merr = (np.abs(gmin - dsel) / np.maximum(dsel, 1e-30)).max()
    print("n=%d d=%d k=%d: mismatches=%d worst_rel_margin=%.3g sums_err=%.3g cnt_err=%d min_rel_err=%.3g inertia=%.9g want=%.9g"
          % (n, d, k, len(bad), worst, serr, cerr, merr, inertia.item(), omin.sum()), flush=True)
