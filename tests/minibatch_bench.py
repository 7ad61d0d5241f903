"""Side measurement (not collected by pytest, not the bench contract): PartialMiniBatchKMeans on C2-shaped data
(10M x 64 fp32 blobs, k = 256) in 1M-row blocks, device-resident and host-resident, one JSON line.
    python tests/minibatch_bench.py [--n N] [--reps R]
Per block: the fused E+M kernel time (bkm_lloyd_chunk with FIRST_CHUNK | COUNTS_F64) and the step kernel time
(bkm_minibatch_step), CUDA events over R launches after a warm-up; the latency of the step's one host read (k weight
sums and the batch inertia, device idle).  Then whole fits (each block read once), with: the host k-means++
initialisation; the host time of each step after its read returned (the reassignment on reassignment steps, the relabel
on the last block), split into reassignment steps and the others; the time of the O(batch) permutation
``choice(replace=False)`` of scikit-learn's RNG stream and its share; one Lloyd iteration of KMeans over the same data
alongside.  A third arm raises reassignment_ratio so that the reassignment path runs.  The card's name, power limit and
median SM clock are part of the record.
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from bench import ClockSampler, synth_blobs_device
from dask_ml_b200.chunked import ChunkedArray
from dask_ml_b200.cluster import PartialMiniBatchKMeans, k_means as km
from dask_ml_b200.cluster import minibatch as mbm
from dask_ml_b200.engine import Comm, CudaBackend, DeviceData, host_resident


def _arg(name, default):
    return type(default)(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def _kernel_times(be, x, k, reps):
    d = int(x.shape[1])
    C = x[:k].double().contiguous()
    st = mbm._MiniBatchState(be, C.cpu().numpy(), np.zeros(k), torch.float32)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    t_em, t_st = [], []
    for r in range(reps + 2):
        ev[0].record()
        be.lloyd_chunk(x, st.pack, k, None, None, st.sums, st.counts, st.inertia, first=True)
        ev[1].record()
        be.minibatch_step(st.red, st.Cb[st.cur], st.Wb[st.cur], st.Cb[st.cur ^ 1], st.Wb[st.cur ^ 1], st.pack,
                          torch.float32)
        ev[2].record()
        torch.cuda.synchronize()
        if r >= 2:
            t_em.append(ev[0].elapsed_time(ev[1]))
            t_st.append(ev[1].elapsed_time(ev[2]))
    return float(np.median(t_em)), float(np.median(t_st)), d


class _HostTimer(object):
    """Per step: the host time after the step's read returned (the reassignment and, on the last block, the relabel),
    and whether the step reassigned centres."""

    def __init__(self):
        self.t, self.reassigned = [], []
        self._fr = mbm._MiniBatchState.finish_read
        self._end = PartialMiniBatchKMeans._step_end
        timer = self

        def finish_read(st):
            out = timer._fr(st)
            timer.t0 = time.perf_counter()
            return out

        def step_end(est, *a, **k):
            before = est.random_state.reassignments
            out = timer._end(est, *a, **k)
            timer.t.append(time.perf_counter() - timer.t0)
            timer.reassigned.append(est.random_state.reassignments > before)
            return out
        mbm._MiniBatchState.finish_read = finish_read
        PartialMiniBatchKMeans._step_end = step_end

    def close(self):
        mbm._MiniBatchState.finish_read = self._fr
        PartialMiniBatchKMeans._step_end = self._end


class _CountingRandomState(np.random.RandomState):
    """Counts and times the reassignment draws (``choice`` without replacement and weights: the O(batch) permutation
    of scikit-learn's RNG stream)."""

    def __init__(self, seed):
        super().__init__(seed)
        self.reassignments = 0
        self.permutation_s = []

    def choice(self, a, size=None, replace=True, p=None):
        if replace or p is not None:
            return super().choice(a, size=size, replace=replace, p=p)
        t = time.perf_counter()
        out = super().choice(a, size=size, replace=replace, p=p)
        self.permutation_s.append(time.perf_counter() - t)
        self.reassignments += 1
        return out


def _fit_time(X, k, seed, ratio):
    # default batch_size (1024): k-means++ runs on the host over init_size = 3 * 1024 rows of the first block, and
    # the reassignment check runs every third block (10 * k rows counted at 1024 per step)
    est = PartialMiniBatchKMeans(n_clusters=k, random_state=_CountingRandomState(0), reassignment_ratio=ratio)
    init = PartialMiniBatchKMeans._init_centroids_host
    t_init = []

    def timed_init(self, *a):
        t = time.perf_counter()
        out = init(self, *a)
        t_init.append(time.perf_counter() - t)
        return out
    PartialMiniBatchKMeans._init_centroids_host = timed_init
    np.random.seed(seed)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    try:
        est.fit(X)
        est.labels_.blocks[0].cpu()
        torch.cuda.synchronize()
    finally:
        PartialMiniBatchKMeans._init_centroids_host = init
    return time.perf_counter() - t0, est, t_init[0]


def _lloyd_time(X, centers):
    st = km.LloydState(X, centers)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    km.lloyd_loop(st, 1, 0.0)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def _read_ms(be, k, reps):
    """The step's one host read (k weight sums + the batch inertia) with the device idle: its own latency."""
    st = mbm._MiniBatchState(be, np.zeros((k, 64)), np.zeros(k), torch.float32)
    t = []
    for _ in range(reps + 5):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        st.start_read()
        st.finish_read()
        t.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(t[5:]))


def _ms(v, f=np.median):
    return 1e3 * float(f(v)) if len(v) else None


def main():
    import warnings

    warnings.simplefilter("ignore", FutureWarning)
    n, d, k, rows, reps = _arg("--n", 10_000_000), 64, 256, 1 << 20, _arg("--reps", 20)
    be = CudaBackend()
    dev = be.device
    Xall = synth_blobs_device(n, d, 256, 7, dev, torch.float32)
    blocks = [Xall[s:s + rows] for s in range(0, n, rows)]
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    t_em, t_step, _ = _kernel_times(be, blocks[0], k, reps)
    rec = {"shape": "C2-shaped %d x %d fp32 blobs, k=%d, %d-row blocks (%d blocks)" % (n, d, k, rows, len(blocks)),
           "per_block": {"em_kernel_ms": t_em, "step_kernel_ms": t_step, "host_read_ms": _read_ms(be, k, 200)}}
    host = Xall.cpu()
    del Xall
    Xh = host_resident(ChunkedArray([host[s:s + rows] for s in range(0, n, rows)]), be, block_rows=rows)
    Xd = DeviceData(blocks, be, Comm())
    # reassignment_ratio 0.3: the centres k-means++ put two to a blob hold about half a blob each and are reassigned
    # at the checks (every third step), so the host reassignment path and its permutation of 1M indices are timed
    for name, X, ratio in (("resident", Xd, 0.01), ("host_resident", Xh, 0.01), ("resident_reassign", Xd, 0.3)):
        _fit_time(X, k, 1, ratio)                                  # warm-up (init, every kernel shape)
        timer = _HostTimer()
        try:
            fits = [_fit_time(X, k, 2 + r, ratio) for r in range(3)]
        finally:
            timer.close()
        est = fits[-1][1]
        lloyd = [_lloyd_time(X, est.cluster_centers_) for _ in range(3)]
        fit_s = float(np.median([f[0] for f in fits]))
        re = [t for t, r in zip(timer.t, timer.reassigned) if r]
        other = [t for t, r in zip(timer.t, timer.reassigned) if not r]
        perm = [t for f in fits for t in f[1].random_state.permutation_s]
        rec[name] = {"reassignment_ratio": ratio, "fit_s": fit_s, "lloyd_iteration_s": float(np.median(lloyd)),
                     "host_init_s": float(np.median([f[2] for f in fits])),
                     "reassignment_steps_per_fit": [f[1].random_state.reassignments for f in fits],
                     "steps_per_fit": len(blocks),
                     "host_after_read_ms_other_steps_median": _ms(other), "host_after_read_ms_other_steps_max": _ms(other, np.max),
                     "host_after_read_ms_reassign_steps_median": _ms(re),
                     "permutation_ms_median": _ms(perm),
                     "permutation_share_of_reassign_step_host_time": (float(np.sum(perm) / np.sum(re)) if re else None),
                     "permutation_share_of_fit": float(np.sum(perm) / (3 * fit_s))}
    clocks = sampler.stop()
    clocks["gpu"] = torch.cuda.get_device_name(dev)
    rec["device"] = clocks
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
