"""Side measurements (not collected by pytest, not the bench contract): Lloyd-iteration time of single BASELINE.json
shapes on one GPU against their HBM roofline (algorithmic bytes d*s+4 per sample).  Used as the short command under ncu.
    python tests/shape_bench.py [C3 C4 C1 C2simt ...] [--steps K]
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from bench import synth_blobs_device, synth_config_device
from dask_ml_b200.cluster.k_means import LloydState
from dask_ml_b200.engine import Comm, CudaBackend, DeviceData

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
peaks = json.load(open(pk)) if os.path.exists(pk) else {"hbm_gbs": 6650.0}
SHAPES = {
    "C3": ("C3 KDD-shaped 4.9M x 41 f32 k=100", 4_898_431, 41, 100, torch.float32, 0),
    "C4": ("C4 airline-shaped shard 15M x 13 f32 k=20 (1/8 of 120M)", 15_000_000, 13, 20, torch.float32, 0),
    "C4pad": ("C4 with a 16-float row pitch", 15_000_000, 13, 20, torch.float32, 0),
    "C1": ("C1 100k x 16 f64 k=8", 100_000, 16, 8, torch.float64, 0),
    "C2": ("C2 10M x 64 f32 k=256", 10_000_000, 64, 256, torch.float32, 0),
    "C2simt": ("C2 on the generic CUDA-core kernel (FORCE_SIMT) 2M x 64 f32 k=256", 2_000_000, 64, 256, torch.float32, 1),
    "C4simt": ("C4 on the generic CUDA-core kernel (FORCE_SIMT)", 15_000_000, 13, 20, torch.float32, 1),
    # family 2 with k = 25..32, which runs on the one-row-per-thread streaming kernel (k <= 24: two rows per thread)
    "F2d15k32": ("family 2, 15M x 15 f32 k=32", 15_000_000, 15, 32, torch.float32, 0),
    "F2d16k28": ("family 2, 15M x 16 f32 k=28", 15_000_000, 16, 28, torch.float32, 0),
    "F2d12k32": ("family 2, 15M x 12 f32 k=32", 15_000_000, 12, 32, torch.float32, 0),
    "F2d8k32": ("family 2, 15M x 8 f32 k=32", 15_000_000, 8, 32, torch.float32, 0),
    "F2d4k30": ("family 2, 15M x 4 f32 k=30", 15_000_000, 4, 30, torch.float32, 0),
}
args = [a for a in sys.argv[1:] if not a.startswith("--")]
steps = 10
if "--steps" in sys.argv:
    steps = int(sys.argv[sys.argv.index("--steps") + 1])
    args = [a for a in args if a != str(steps)]
names = args or ["C3", "C4", "C4pad", "C1", "C2simt"]
be = CudaBackend()
for key in names:
    name, n, d, k, dt, flags = SHAPES[key]
    be.flags = flags
    base = key.replace("pad", "").replace("simt", "")
    if base in ("C3", "C4"):
        X = synth_config_device(base, n, 0, be.device)
    else:
        X = synth_blobs_device(n, d, k, 7, be.device, dt)
    if key == "C4pad" or (d % 4 and be.kernel_family(d, k, dt) == 1):
        X = be.to_device(X, dt)          # padded row pitch (16-byte rows)
    data = DeviceData([X], be, Comm())
    st = LloydState(data, X[:k].cpu().numpy().astype(np.float64))
    for _ in range(3):
        st.step(); st.accept()
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        st.step(); st.accept()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    s = 4 if dt == torch.float32 else 8
    gbs = n * (d * s + 4) / (ms * 1e-3) / 1e9
    tf = 2.0 * n * d * k / (ms * 1e-3) / 1e12
    rec = {"shape": name, "kernel_family": int(be.kernel_family(d, k, dt)), "row_pitch": int(X.stride(0)), "ms_per_iter": ms,
           "samples_per_s": n / (ms * 1e-3), "hbm_gbs": gbs, "hbm_frac_of_measured": gbs / peaks["hbm_gbs"], "tflops": tf}
    print(json.dumps(rec), flush=True)
    del X, data, st
    torch.cuda.empty_cache()
