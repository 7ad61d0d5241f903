"""Times the four passes of PartialMultinomialNB / PartialBernoulliNB on the device against the float64 torch
composition of the same arithmetic (alternated in the same process) and against scikit-learn's ``partial_fit`` /
``predict`` on the CPU for the same block.

    python tests/partial_nb_bench.py [--reps R] [--out FILE]

Workloads: 2^20 x 1000 fp32 counts with K = 20; 2^20 x 256 fp32 counts with K = 200; hashed CSR 262144 x 2^20 with
about 100 nonzeros per row and K = 20 (the SGD bench's text shape).  Every device time is the median of R CUDA-event
timings after a warm-up call; the HBM floor is the bytes the pass must move over 3.35 TB/s."""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from sklearn import naive_bayes as sknb  # noqa: E402

from dask_ml_b200.engine import CudaBackend  # noqa: E402

warnings.simplefilter("ignore")
HBM = 3.35e12


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                     text=True).strip().splitlines()[0]
    except Exception:
        pl = "unknown"
    return name, pl


def _median_ms(fns, reps):
    """Median CUDA-event time of each callable, the callables alternated within every repetition."""
    for f in fns:
        f()
    times = [[] for _ in fns]
    for _ in range(reps):
        for i, f in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            times[i].append(a.elapsed_time(b))
    return [float(np.median(t)) for t in times]


def _host_s(f):
    t0 = time.perf_counter()
    f()
    return time.perf_counter() - t0


def dense(be, n, d, K, reps, seed):
    rng = np.random.RandomState(seed)
    Xh = rng.poisson(0.5, size=(n, d)).astype(np.float32)
    yh = rng.randint(0, K, size=n)
    x = torch.from_numpy(Xh).cuda()
    cls = torch.from_numpy(yh.astype(np.int32)).cuda()
    fc, cc = be.empty((K, d), torch.float64), be.empty((K,), torch.float64)
    sk = sknb.MultinomialNB()
    fit_s = _host_s(lambda: sk.partial_fit(Xh, yh, classes=np.arange(K)))
    W = torch.from_numpy(sk.feature_log_prob_).cuda()
    b = torch.from_numpy(sk.class_log_prior_).cuda()
    lab = be.empty((n,), torch.int32)
    out = be.empty((n, K), torch.float64)
    idx = cls.long()

    def torch_counts():
        f = torch.zeros((K, d), dtype=torch.float64, device="cuda")
        f.index_add_(0, idx, x.double())
        torch.bincount(idx, minlength=K)

    def torch_jll():
        return x.double() @ W.T + b

    ours = _median_ms([lambda: be.class_counts_chunk(x, cls, K, fc, cc, first=True), torch_counts], reps)
    pl = _median_ms([lambda: be.nb_linear_jll_chunk(x, W, b, labels=lab),
                     lambda: torch_jll().argmax(dim=1)], reps)
    pp = _median_ms([lambda: be.nb_linear_jll_chunk(x, W, b, out=out, out_mode=1),
                     lambda: torch.log_softmax(torch_jll(), dim=1)], reps)
    ok = bool((fc.cpu().numpy() == sk.feature_count_).all())
    agree = float((lab.cpu().numpy() == torch_jll().argmax(dim=1).cpu().numpy()).mean())
    pred_s = _host_s(lambda: sk.predict(Xh))
    xb = n * d * 4
    return dict(workload="dense %dx%d fp32 counts, K=%d" % (n, d, K),
                counts=dict(ms=ours[0], torch_ms=ours[1], floor_ms=1e3 * (xb + n * 4) / HBM, exact=ok),
                predict_labels=dict(ms=pl[0], torch_ms=pl[1], floor_ms=1e3 * (xb + n * 4) / HBM,
                                    label_agreement_with_torch=agree),
                predict_log_proba=dict(ms=pp[0], torch_ms=pp[1], floor_ms=1e3 * (xb + n * K * 8) / HBM),
                sklearn_partial_fit_s=fit_s, sklearn_predict_s=pred_s)


def hashed(be, n, nnz, K, reps, seed):
    rng = np.random.RandomState(seed)
    d = 1 << 20
    cols = np.sort(np.stack([rng.choice(d, nnz, replace=False) for _ in range(64)]), axis=1)
    cols = cols[np.arange(n) % 64]
    vals = rng.randint(1, 4, size=(n, nnz)).astype(np.float64)
    A = sp.csr_matrix((vals.ravel(), cols.ravel(), np.arange(0, n * nnz + 1, nnz)), shape=(n, d))
    yh = rng.randint(0, K, size=n)
    blk = (torch.from_numpy(A.indptr.astype(np.int64)).cuda(), torch.from_numpy(A.indices.astype(np.int64)).cuda(),
           torch.from_numpy(A.data).cuda(), n)
    cls = torch.from_numpy(yh.astype(np.int32)).cuda()
    sk = sknb.MultinomialNB()
    fit_s = _host_s(lambda: sk.partial_fit(A, yh, classes=np.arange(K)))
    WT = torch.from_numpy(np.ascontiguousarray(sk.feature_log_prob_.T)).cuda()
    b = torch.from_numpy(sk.class_log_prior_).cuda()
    fcT = be.empty((d, K), torch.float64)
    lab = be.empty((n,), torch.int32)
    out = be.empty((n, K), torch.float64)
    Xt = torch.sparse_csr_tensor(blk[0], blk[1], blk[2], size=(n, d))
    rows = torch.repeat_interleave(torch.arange(n, device="cuda"), blk[0][1:] - blk[0][:-1])
    lin = cls.long()[rows] * d + blk[1]

    def ours_counts():
        csc = be.csr_transpose_chunk(blk, d)
        be.csc_class_counts_chunk(csc, d, cls, K, fcT, first=True)

    def torch_counts():
        f = torch.zeros(K * d, dtype=torch.float64, device="cuda")
        f.index_add_(0, lin, blk[2])

    c = _median_ms([ours_counts, torch_counts], reps)
    pl = _median_ms([lambda: be.nb_csr_jll_chunk(blk, d, WT, b, labels=lab),
                     lambda: (torch.sparse.mm(Xt, WT) + b).argmax(dim=1)], reps)
    pp = _median_ms([lambda: be.nb_csr_jll_chunk(blk, d, WT, b, out=out, out_mode=1),
                     lambda: torch.log_softmax(torch.sparse.mm(Xt, WT) + b, dim=1)], reps)
    ok = bool((fcT.cpu().numpy().T == sk.feature_count_).all())
    pred_s = _host_s(lambda: sk.predict(A))
    agree = float((lab.cpu().numpy() == sk.predict(A)).mean())
    nz = n * nnz
    return dict(workload="hashed CSR %dx2^20, %d nonzeros per row, K=%d" % (n, nnz, K),
                counts_with_transpose=dict(ms=c[0], torch_ms=c[1], exact=ok,
                                           floor_ms=1e3 * (nz * 20 + n * 12 + d * K * 8) / HBM),
                predict_labels=dict(ms=pl[0], torch_ms=pl[1], floor_ms=1e3 * (nz * 16 + n * 12) / HBM,
                                    label_agreement_with_sklearn=agree),
                predict_log_proba=dict(ms=pp[0], torch_ms=pp[1], floor_ms=1e3 * (nz * 16 + n * (8 + K * 8)) / HBM),
                sklearn_partial_fit_s=fit_s, sklearn_predict_s=pred_s)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the bench needs a GPU"
    name, pl = _card()
    be = CudaBackend()
    res = dict(card=name, power_limit=pl, reps=args.reps, workloads=[])
    for run in (lambda: dense(be, 1 << 20, 1000, 20, args.reps, 0), lambda: dense(be, 1 << 20, 256, 200, args.reps, 1),
                lambda: hashed(be, 262144, 100, 20, args.reps, 2)):
        r = run()
        print(json.dumps(r), flush=True)
        res["workloads"].append(r)
        torch.cuda.empty_cache()
    print(json.dumps(dict(card=name, power_limit=pl)))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
