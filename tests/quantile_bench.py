"""Speed of QuantileTransformer's passes on one GPU (run on an H100: python tests/quantile_bench.py [--out FILE]).

Shapes: 10M x 64 fp32, 8M x 128 bf16 and 10M x 64 fp64, n_quantiles = 1000 (2000 target ranks per column).
  * fit: CUDA-event times of each selection round (bkm_quantile_hist_chunk + bkm_quantile_select_step) and of the whole
    fit (rounds, state read-back and host interpolation), alternated in the same process with a ``sort(0)``-based
    percentile in torch; the outputs are compared;
  * transform: forward and inverse for both distributions (bkm_quantile_transform_chunk), against the HBM floor of one
    read of X and one 8-byte write per element (3.35 TB/s).
The card's name and power limit come from the same run.
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
from dask_ml_b200.preprocessing.data import RADIX_ROUNDS, quantile_transform, quantiles_exact  # noqa: E402
from nb_bench import PEAK_BW, _card, _pair, _time  # noqa: E402

NQ = 1000


def round_times(be, x, references, reps):
    """Median CUDA-event time of each selection round over ``reps`` fits (one chunk, one column group)."""
    n, d = x.shape
    qf = torch.as_tensor(np.true_divide(references * 100, 100.0)).cuda()
    rounds = RADIX_ROUNDS[x.dtype]
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(rounds + 1)]
    out = []
    for _ in range(reps):
        state = be.quantile_state_new(d, NQ)
        ev[0].record()
        for r in range(rounds):
            h = torch.empty((d * min(2 * NQ, 256 ** r) * 256,), dtype=torch.float64, device="cuda")
            be.quantile_hist_chunk(x, state, NQ, r, h, first=True)
            be.quantile_select_step(h, state, d, NQ, r, x.dtype, qf)
            ev[r + 1].record()
        torch.cuda.synchronize()
        out.append([ev[r].elapsed_time(ev[r + 1]) for r in range(rounds)])
    return [float(v) for v in np.median(np.asarray(out), axis=0)]


def run(n, d, dt, reps):
    be = CudaBackend()
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (torch.randn((n, d), generator=g, device="cuda", dtype=torch.float32) * 2 + 5).to(dt)
    data = DeviceData([x], be)
    references = np.linspace(0, 1, NQ)
    res = {}

    def fused_fit():
        res["f"] = quantiles_exact(data, references)

    def torch_fit():
        srt = x.sort(0).values.double()
        vi = torch.as_tensor(references, dtype=torch.float64).cuda() * (n - 1)
        lo = vi.floor().long()
        hi = torch.clamp(lo + 1, max=n - 1)
        a, b = srt[lo], srt[hi]
        res["t"] = (a + (b - a) * (vi - vi.floor())[:, None]).cpu()

    fused_fit()
    torch_fit()
    torch.cuda.synchronize()
    err_fit = float(np.abs(res["f"] - res["t"].numpy()).max())
    meta = dict(n=n, d=d, dtype=str(dt).replace("torch.", ""), n_quantiles=NQ)
    es = x.element_size()
    rows = [_pair("fit", fused_fit, torch_fit, max(2, reps // 3), RADIX_ROUNDS[dt] * n * d * es,
                  dict(max_abs_vs_sort=err_fit), dict(meta, rounds_ms=round_times(be, x, references, 5)))]
    q = res["f"]
    y = None
    for dist in ("uniform", "normal"):
        def fwd():
            res["y"] = quantile_transform(data, q, references, False, dist)

        fwd()
        y = DeviceData(res["y"].blocks, be)

        def inv():
            res["x"] = quantile_transform(y, q, references, True, dist)

        for name, fn, byts in (("forward", fwd, n * d * (es + 8)), ("inverse", inv, n * d * 16)):
            t = _time(fn, reps)
            rows.append(dict(meta, pass_="transform_%s_%s" % (name, dist), fused_ms=t, gbps=byts / t / 1e6,
                             floor_ms=byts / PEAK_BW * 1e3))
        inv()
        back = res["x"].blocks[0]
        torch.cuda.synchronize()
        rows[-1]["max_abs_round_trip"] = float((back - x.double()).abs().max())
        del y, res["y"], res["x"]
        torch.cuda.empty_cache()
    return rows


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
