"""Side measurement (not collected by pytest, not the bench contract): the two Nystrom passes of SpectralClustering on
C2-shaped data (10M x 64 fp32 blobs), l in {100, 256} keep rows, k = 8, one JSON line.
    python tests/spectral_bench.py [--n N] [--reps R]
Per l: each pass's kernel time (CUDA events, warmed up), its algorithmic rate (2 d l flop per row and pass) and HBM
bytes/s against the H100 SXM data sheet (67 TFLOP/s fp32 CUDA cores, 989 TFLOP/s dense fp16 tensor cores, 3.35 TB/s);
the "blocks" arm built from existing pieces (bkm_transform_chunk mode 2 into an (n, l) buffer, then torch sum and
matmul), alternated with the fused arm in the same process; the whole SpectralClustering.fit.  The card's name, power
limit and median SM clock are part of the record.
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from bench import ClockSampler, synth_blobs_device
from dask_ml_b200.cluster import SpectralClustering
from dask_ml_b200.engine import Comm, CudaBackend, DeviceData

HBM_GBS, FP32_TFLOPS, FP16_TFLOPS = 3350.0, 67.0, 989.0


def _arg(name, default):
    return type(default)(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def main():
    n, d, k, reps = _arg("--n", 10_000_000), 64, 8, _arg("--reps", 5)
    be = CudaBackend()
    dev = be.device
    X = synth_blobs_device(n, d, 256, 7, dev, torch.float32)
    gamma = 1.0 / (2.0 * d)
    rec = {"shape": "C2-shaped %d x %d fp32 blobs, k=%d, gamma=%g" % (n, d, k, gamma), "arms": []}
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    for l in (100, 256):
        keep = X[torch.as_tensor(np.sort(np.random.RandomState(l).choice(n, l, replace=False)), device=dev)]
        pack = be.pack_centers(keep.double().contiguous(), torch.float32)
        W = torch.as_tensor(np.random.RandomState(1).standard_normal((l, k)), dtype=torch.float32, device=dev)
        cs = be.zeros((l,), torch.float64)
        emb = be.zeros((n, k), torch.float32)
        K = be.empty((n, l), torch.float32)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]

        def fused():
            ev[0].record()
            be.kernel_colsum(X, pack, l, gamma, cs, first=True)
            ev[1].record()
            be.nystrom_embed(X, pack, l, gamma, W, emb)
            ev[2].record()

        def blocks():
            ev[0].record()
            be.transform_chunk(X, pack, l, K, mode=2, gamma=gamma)
            c = K.sum(0, dtype=torch.float64)
            e = K @ W
            e = e / torch.sqrt((e * e).sum(1, keepdim=True))
            ev[3].record()
            return c, e

        for _ in range(2):                                          # warm-up of every shape the timed loop uses
            fused(); blocks()
        torch.cuda.synchronize()
        t_cs, t_em, t_fu, t_bl = [], [], [], []
        for _ in range(reps):                                       # the two arms alternate
            fused(); torch.cuda.synchronize()
            t_cs.append(ev[0].elapsed_time(ev[1])); t_em.append(ev[1].elapsed_time(ev[2]))
            t_fu.append(ev[0].elapsed_time(ev[2]))
            blocks(); torch.cuda.synchronize()
            t_bl.append(ev[0].elapsed_time(ev[3]))
        ms = lambda v: float(np.median(v))
        flop = 2.0 * n * d * l
        x_bytes = n * d * 4.0
        arm = {"l": l,
               "colsum_ms": ms(t_cs), "colsum_tflops": flop / ms(t_cs) * 1e-9, "colsum_gbs": x_bytes / ms(t_cs) * 1e-6,
               "embed_ms": ms(t_em), "embed_tflops": flop / ms(t_em) * 1e-9,
               "embed_gbs": (x_bytes + n * k * 4.0) / ms(t_em) * 1e-6,
               "fused_ms": ms(t_fu), "blocks_ms": ms(t_bl),
               "blocks_bytes_extra_gb": 2 * n * l * 4.0 * 1e-9,
               "fused_hbm_roof_ms": (2 * x_bytes + n * k * 4.0) / HBM_GBS * 1e-6}
        del K
        torch.cuda.empty_cache()
        data = DeviceData([X], be, Comm())
        sc = SpectralClustering(n_clusters=k, n_components=l, gamma=gamma, random_state=0)
        sc.fit(data)                                                # warm-up (KMeans kernels, host algebra)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sc.fit(data)
        sc.labels_.blocks[0].cpu()
        torch.cuda.synchronize()
        arm["fit_s"] = time.perf_counter() - t0
        arm["fit_kmeans_n_iter"] = int(sc.assign_labels_.n_iter_)
        rec["arms"].append(arm)
    clocks = sampler.stop()
    clocks["gpu"] = torch.cuda.get_device_name(dev)
    rec["device"] = clocks
    rec["roofs"] = {"hbm_gbs": HBM_GBS, "fp32_tflops": FP32_TFLOPS, "fp16_dense_tflops": FP16_TFLOPS}
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
