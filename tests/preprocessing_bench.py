"""Speed of the scalers' passes on one GPU (run on an H100: python tests/preprocessing_bench.py [--out FILE]).

Shapes: 10M x 64 fp32, 8M x 128 bf16 and 10M x 64 fp64.  CUDA-event times of each pass, alternated in the same process
with the torch composition it replaces, and the outputs compared:
  * statistics (bkm_colstats_chunk) against ``X.double()`` then mean, var, amin and amax over rows;
  * transform (bkm_affine_chunk, (x - m) / s in X's dtype, float32 for bf16) against ``(X - m) / s`` in torch;
  * percentiles (RobustScaler's 25 / 50 / 75, every radix round and the host interpolation) against a
    ``sort(0)``-based percentile.
GB/s count one read of X for the statistics, one read and one write for the transform and one read per radix round for
the percentiles, against the HBM floor (3.35 TB/s).  The card's name and power limit come from the same run.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from dask_ml_b200.engine import CudaBackend, DeviceData  # noqa: E402
from dask_ml_b200.preprocessing.data import RADIX_ROUNDS, percentiles  # noqa: E402
from nb_bench import _card, _pair  # noqa: E402

Q = [25, 50.0, 75]


def run(n, d, dt, reps):
    be = CudaBackend()
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (torch.randn((n, d), generator=g, device="cuda", dtype=torch.float32) * 2 + 5).to(dt)
    odt = torch.float32 if dt == torch.bfloat16 else dt
    es, eo = x.element_size(), torch.empty((), dtype=odt).element_size()
    shift = x[:1024].double().mean(0)
    acc = torch.empty((5, d), dtype=torch.float64, device="cuda")
    mm = torch.empty((2, d), dtype=torch.float64, device="cuda")
    m = torch.randn((d,), generator=g, device="cuda", dtype=torch.float64).to(odt)
    s = (torch.rand((d,), generator=g, device="cuda", dtype=torch.float64) + 0.5).to(odt)
    out = be.rows_buffer(n, d, odt)
    data = DeviceData([x], be)
    res = {}

    def fused_stats():
        be.colstats_chunk(x, shift, acc, mm, first=True)

    def torch_stats():
        xd = x.double()
        res["t_stats"] = (xd.mean(0), xd.var(0, unbiased=False), xd.amin(0), xd.amax(0))

    def fused_affine():
        be.affine_chunk(x, m.double(), s.double(), 1, 1, out)

    def torch_affine():
        res["t_aff"] = (x.to(odt) - m) / s

    def fused_pct():
        res["f_pct"] = percentiles(data, Q)

    def torch_pct():
        srt = x.sort(0).values.double()
        qf = torch.tensor(Q, dtype=torch.float64) / 100 * (n - 1)
        lo, fr = qf.floor().long(), qf - qf.floor()
        hi = torch.clamp(lo + 1, max=n - 1)
        a, b = srt[lo.cuda()], srt[hi.cuda()]
        res["t_pct"] = (a + (b - a) * fr.cuda()[:, None]).T

    for f in (fused_stats, torch_stats, fused_affine, torch_affine, fused_pct, torch_pct):
        f()
    torch.cuda.synchronize()
    n_ = acc.new_tensor(float(n))
    mean = shift + acc[0] / n_
    var = acc[1] / n_ - (acc[0] / n_) ** 2
    tm, tv, tlo, thi = res["t_stats"]
    err_stats = dict(mean=float(((mean - tm).abs() / tm.abs()).max()), var=float(((var - tv).abs() / tv).max()),
                     minmax=float(max((mm[0] - tlo).abs().max(), (mm[1] - thi).abs().max())))
    err_aff = float((out.to(torch.float64) - res["t_aff"].to(torch.float64)).abs().max())
    err_pct = float(np.abs(res["f_pct"] - res["t_pct"].cpu().numpy()).max())
    meta = dict(n=n, d=d, dtype=str(dt).replace("torch.", ""))
    xb = n * d * es
    return [
        _pair("colstats", fused_stats, torch_stats, reps, xb, err_stats, meta),
        _pair("affine", fused_affine, torch_affine, reps, xb + n * d * eo, dict(max_abs=err_aff), meta),
        _pair("percentiles", fused_pct, torch_pct, max(2, reps // 3), RADIX_ROUNDS[dt] * xb, dict(max_abs=err_pct),
              dict(meta, rounds=RADIX_ROUNDS[dt])),
    ]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    card = _card()
    rows = []
    for n, d, dt in ((10_000_000, 64, torch.float32), (8_000_000, 128, torch.bfloat16), (10_000_000, 64, torch.float64)):
        rows += run(n, d, dt, args.reps)
        torch.cuda.empty_cache()
    for r in rows:
        print(json.dumps(r))
    print("card:", card)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": card, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
