"""The C-ABI boundary on the CPU: every ``CudaBackend`` kernel method, the device paths of ``datasets`` and the SGD row
orders run against a fake ``libbkm_b200.so`` that checks each call against its ``_lib.SIGNATURES`` prototype (argument
count, and every argument through its declared argtype's ``from_param``) and records it.  The record must equal
``tests/golden/backend_calls.json``, so a change to the Python side of the boundary that alters any argument of any call
fails here without a GPU.

The record names pointers by what they point at: a tensor or array this file made (``name`` or ``name+<byte offset>``
for a view), a backend scratch buffer (``ws:<key>``), the current stream (``stream``), a buffer the method allocated
and returned (``<step>:<i>``), or ``new`` for one it allocated and dropped.  A ``byref`` struct is recorded as its
fields, a host array as its values, a size query's output as ``out``.

``python tests/test_backend_calls_host.py --record`` rewrites the golden from the code in the tree."""
import ctypes
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from dask_ml_b200 import _lib, datasets, engine  # noqa: E402
from dask_ml_b200.linear_model import _sgd  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "backend_calls.json")
STREAM = 0x5EA0
# host-only, debug and peer-memory entry points: no CudaBackend kernel method has to reach them
NOT_DRIVEN = ("bkm_version", "bkm_error_string", "bkm_device_info", "bkm_p2p_", "bkm_allreduce_p2p", "bkm_debug_",
              "bkm_launch_count")
_SIZES = {name: 4096 + 512 * i for i, name in enumerate(sorted(n for n in _lib.SIGNATURES if n.endswith("_bytes")))}
_SIZE_P = ctypes.POINTER(ctypes.c_size_t)


class _Stream(object):
    cuda_stream = STREAM


class _Device(object):
    """Stands in for ``torch.cuda.device``: no device switch, but the record notes whether a call ran inside one."""

    depth = 0

    def __init__(self, device):
        pass

    def __enter__(self):
        _Device.depth += 1

    def __exit__(self, *exc):
        _Device.depth -= 1


class _FakeFn(object):
    def __init__(self, lib, name, restype, argtypes):
        self.lib, self.name, self.restype, self.argtypes = lib, name, restype, argtypes

    def __call__(self, *args):
        name = self.name
        assert len(args) == len(self.argtypes), "%s takes %d arguments, got %d" % (name, len(self.argtypes), len(args))
        for i, (a, t) in enumerate(zip(args, self.argtypes)):
            try:
                t.from_param(a)
            except Exception as e:
                raise AssertionError("%s argument %d (%r) does not convert to %s: %s" % (name, i, a, t.__name__, e))
        outs = 0
        for a, t in zip(args, self.argtypes):
            if t is _SIZE_P:
                a._obj.value = _SIZES[name] + 128 * outs        # distinct sizes, also for a second output
                outs += 1
        self.lib.calls.append([name, _Device.depth > 0, [self._raw(a, t) for a, t in zip(args, self.argtypes)]])
        if self.restype is None:
            return None
        return b"fake" if self.restype is ctypes.c_char_p else 0

    @staticmethod
    def _raw(a, t):
        if t is ctypes.c_void_p:
            if isinstance(a, ctypes.c_void_p):
                held = [o for o in (a._objects or {}).values() if isinstance(o, ctypes.Array)]
                if held:
                    return {"host": list(held[0])}
                a = a.value
            return ("ptr", a or 0)
        if issubclass(t, ctypes._Pointer):                                          # byref(...)
            obj = a._obj
            if isinstance(obj, ctypes.Structure):
                return {f: getattr(obj, f) for f, _ in obj._fields_}
            return "out"
        return a.value if isinstance(a, ctypes._SimpleCData) else a


class _FakeLib(object):
    """Answers every name of ``_lib.SIGNATURES``."""

    def __init__(self):
        self.calls = []
        for name, (res, argtypes) in _lib.SIGNATURES.items():
            setattr(self, name, _FakeFn(self, name, res, argtypes))


class _Recorder(object):
    """Runs the steps and resolves each call's pointers once its step has returned."""

    def __init__(self, lib, be):
        self.lib, self.be = lib, be
        self.named = []                    # (name, base address, bytes)
        self.alive = []                    # the named tensors, kept so that no later buffer reuses their addresses
        self.log = []

    def name(self, name, obj):
        self.alive.append(obj)
        self.named.append((name, obj.data_ptr(), obj.numel() * obj.element_size()))
        return obj

    def t(self, name, shape, dtype=torch.float64):
        return self.name(name, torch.zeros(shape, dtype=dtype))

    def _where(self, p, ranges):
        for name, lo, nb in ranges:
            if p == lo or lo <= p < lo + nb:
                return name if p == lo else "%s+%d" % (name, p - lo)
        return None

    def _resolve(self, v, returned):
        if not (isinstance(v, tuple) and v[0] == "ptr"):
            return v
        p = v[1]
        if p == 0:
            return None
        if p == STREAM:
            return "stream"
        ws = [("ws:" + k, b.data_ptr(), b.numel()) for k, b in self.be._ws.items()]
        return self._where(p, ws) or self._where(p, self.named) or self._where(p, returned) or "new"

    def step(self, label, fn, *args, **kw):
        del self.lib.calls[:]
        ret = fn(*args, **kw)
        flat = list(ret) if isinstance(ret, (tuple, list)) else [ret]
        blocks = []
        for r in flat:
            blocks.extend(r.blocks if isinstance(r, datasets.ChunkedArray) else [r])
        returned = []
        for i, r in enumerate(blocks):
            if isinstance(r, torch.Tensor):
                returned.append(("%s:%d" % (label, i), r.data_ptr(), r.numel() * r.element_size()))
            elif isinstance(r, np.ndarray):
                returned.append(("%s:%d" % (label, i), r.ctypes.data, r.nbytes))
        for name, dev, raw in self.lib.calls:
            self.log.append([label, name, dev, [self._resolve(v, returned) for v in raw]])
        return ret


def _drive(rec, be):
    """Every public kernel method of CudaBackend, each mode branch, first / not first, zero-row blocks."""
    t, s = rec.t, rec.step
    f32, f64, i32, i64, u8 = torch.float32, torch.float64, torch.int32, torch.int64, torch.uint8
    n, d, k = 6, 5, 3
    x = rec.name("x", torch.zeros((n, d), dtype=f32))
    x64 = rec.name("x64", torch.zeros((n, d), dtype=f64))
    xbf = rec.name("xbf", torch.zeros((n, d), dtype=torch.bfloat16))
    xpad = rec.name("xpad", torch.zeros((n, 8), dtype=f32))[:, :d]       # row pitch 8
    x0 = rec.name("x0", torch.zeros((0, d), dtype=f32))
    xi = rec.name("xi", torch.zeros((n, 2), dtype=i64))
    pack, labels, min_d2 = t("pack", 512, u8), t("labels", n, i32), t("min_d2", n, f32)
    sums, counts, counts_i, inertia = t("sums", k * d), t("counts", k), t("counts_i", k, i64), t("inertia", 1)
    loop = t("loop", 64, u8)
    s("check_finite", be.check_finite, [x, xpad, xpad[:0]])
    C64 = t("C64", (k, d))
    s("pack_centers/new", be.pack_centers, C64, f32)
    s("pack_centers/out", be.pack_centers, C64, f32, out=t("pack_big", 1 << 16, u8))
    s("lloyd/first", be.lloyd_chunk, x, pack, k, labels, min_d2, sums, counts, inertia, first=True, loop_state=loop)
    s("lloyd/next", be.lloyd_chunk, xpad, pack, k, labels, min_d2, sums, counts_i, inertia)
    s("lloyd/rows0", be.lloyd_chunk, x0, pack, k, labels, min_d2, sums, None, inertia, first=True)
    s("lloyd/bf16", be.lloyd_chunk, xbf, pack, k, labels, min_d2, sums, counts, inertia)
    s("deferred_rows", be.deferred_rows, n, d, k, f32)
    s("kernel_family", be.kernel_family, d, k, f32)
    s("launch_count", be.launch_count)
    s("abort_code", be.abort_code)
    s("reset_abort", be.reset_abort)
    s("loop_state_new", be.loop_state_new, 1e-4, 7)
    red, c_out, state = t("red", k * d + k + 1), t("c_out", (k, d)), t("state", 64, u8)
    s("finalize_step", be.finalize_step, red, C64, c_out, state, pack, f32)
    w_in, w_out = t("w_in", k), t("w_out", k)
    s("minibatch_step", be.minibatch_step, red, C64, w_in, c_out, w_out, pack, f64)
    s("assign", be.assign_chunk, x, pack, k, labels, min_d2, True, inertia)
    s("assign/rows0", be.assign_chunk, x0, pack, k, labels, min_d2, False, None)
    s("sample", be.sample_chunk, min_d2, 0.5, (1 << 64) + 7, 12, t("picked", 4, i64), t("n_picked", 1, i64))
    s("min_fold", be.min_fold, min_d2, t("new_min", n, f32), inertia)
    s("min_fold/none", be.min_fold, min_d2, None, inertia)
    out_nk = t("out_nk", (n, 8), f32)
    s("transform", be.transform_chunk, x, pack, k, out_nk[:, 2:5], 2, 0.25)
    s("transform/rows0", be.transform_chunk, x0, pack, k, out_nk[:0], 0)
    colsum = t("colsum", k)
    s("kernel_colsum/first", be.kernel_colsum, x, pack, k, 0.5, colsum, first=True)
    s("kernel_colsum/next", be.kernel_colsum, x, pack, k, 0.5, colsum)
    shift, csum, gram = t("shift", d), t("csum", d), t("gram", (d, d))
    s("gram/first", be.gram_chunk, x64, shift, csum, gram, first=True)
    s("gram/next", be.gram_chunk, x, None, csum, gram)
    W, colmax = t("W", (k, d)), t("colmax", (k, 4))
    s("project/colmax", be.project_chunk, x, shift, W, colmax=colmax, row_offset=40)
    s("project/out", be.project_chunk, x, None, W, out=t("pout", (n, 4), f32)[:, :k])
    s("project/both", be.project_chunk, x64, shift, W, out=t("pout64", (n, k)), colmax=colmax)
    s("project/rows0", be.project_chunk, x0, shift, W, out=t("pout0", (0, k)))
    s("colmax_new", be.colmax_new, k)
    K = 4
    cls, nbsums, nbcounts, theta = t("cls", n, i32), t("nbsums", (K, d)), t("nbcounts", K), t("theta", (K, d))
    s("class_moments/first", be.class_moments_chunk, x, cls, K, nbsums, nbcounts, first=True)
    s("class_moments/theta", be.class_moments_chunk, x64, cls, K, nbsums, theta=theta)
    inv, logc, jll = t("inv_sigma", (K, d)), t("logc", K), t("jll", (n, K))
    s("nb_jll/labels", be.nb_jll_chunk, x, theta, inv, logc, labels=labels, n_deferred=t("ndef", 1, i32))
    s("nb_jll/out", be.nb_jll_chunk, x, theta, inv, logc, out=jll, exp_out=True)
    s("nb_jll/rows0", be.nb_jll_chunk, x0, theta, inv, logc, out=jll[:0])
    wrow = t("wrow", n)
    s("class_counts/first", be.class_counts_chunk, x, cls, K, nbsums, nbcounts, first=True)
    s("class_counts/w_bin", be.class_counts_chunk, x, cls, K, nbsums, nbcounts, w=wrow, binarize=0.5)
    blk = (t("crow", n + 1, i64), t("col", 10, i64), t("val", 10, f32), n)
    blk64 = (blk[0], blk[1], t("val64", 10), n)
    blk0 = (t("crow0", 1, i64), t("col0", 0, i64), t("val0", 0, f32), 0)
    csc = (t("colptr", d + 1, i64), t("rows", 10, i32), t("vals", 10, f32), t("plan", 8, i64))
    fcT = t("fcT", (d, K))
    s("csc_class_counts/first", be.csc_class_counts_chunk, csc, d, labels, K, fcT, first=True)
    s("csc_class_counts/w_bin", be.csc_class_counts_chunk, csc, d, labels, K, fcT, w=wrow, binarize=0.0)
    Wnb, bnb = t("Wnb", (K, d)), t("bnb", K)
    s("nb_linear_jll/labels", be.nb_linear_jll_chunk, x, Wnb, bnb, labels=labels, binarize=0.0)
    s("nb_linear_jll/out", be.nb_linear_jll_chunk, x, Wnb, bnb, out=jll, out_mode=2)
    s("nb_linear_jll/rows0", be.nb_linear_jll_chunk, x0, Wnb, bnb, out=jll[:0], out_mode=1)
    WT = t("WT", (d, K))
    s("nb_csr_jll/labels", be.nb_csr_jll_chunk, blk, d, WT, bnb, labels=labels, binarize=0.5)
    s("nb_csr_jll/out", be.nb_csr_jll_chunk, blk64, d, WT, bnb, out=jll, out_mode=1)
    s("nb_csr_jll/rows0", be.nb_csr_jll_chunk, blk0, d, WT, bnb, out=jll[:0])
    y, beta, grad, hrow = t("y", n), t("beta", d + 1), t("grad", d + 2), t("hrow", d + 1)
    mu, yes = t("mu", n), t("yes", n, u8)
    s("glm/mode0", be.glm_pass_chunk, x, y, beta, 0, 0, grad=grad, first=True)
    s("glm/mode1", be.glm_pass_chunk, x64, y, beta, 2, 1, grad=grad, hrow=hrow, w=wrow)
    s("glm/mode2", be.glm_pass_chunk, x, None, beta, 1, 2, out=mu)
    s("glm/mode3", be.glm_pass_chunk, x0, None, beta, 0, 3, out=yes[:0])
    s("gram_weighted/first", be.gram_weighted_chunk, x, wrow, gram, first=True)
    s("gram_weighted/next", be.gram_weighted_chunk, x64, wrow, gram)
    r = t("r", n)
    s("glm_csr/mode0", be.glm_csr_pass_chunk, blk, d, y, beta, 0, 0, r=r, grad=grad, first=True)
    s("glm_csr/mode1", be.glm_csr_pass_chunk, blk64, d, y, beta, 2, 1, r=r, w=wrow, grad=grad, hrow=hrow)
    s("glm_csr/mode2", be.glm_csr_pass_chunk, blk, d, None, beta, 1, 2, out=mu)
    s("glm_csr/mode3", be.glm_csr_pass_chunk, blk0, d, None, beta, 0, 3, out=yes[:0])
    s("csr_transpose", be.csr_transpose_chunk, blk, d)
    s("csr_transpose/rows0", be.csr_transpose_chunk, blk0, d)
    v1, o1, v2, o2 = t("v1", n), t("o1", d + 2), t("v2", n), t("o2", d + 1)
    s("csc_matvec/first", be.csc_matvec_chunk, csc, d, v1, o1, first=True)
    s("csc_matvec/two", be.csc_matvec_chunk, csc, d, v1, o1, v2, o2)
    s("gram_weighted_csr/first", be.gram_weighted_csr_chunk, blk, csc, d, wrow, gram, 9, first=True)
    s("gram_weighted_csr/next", be.gram_weighted_csr_chunk, blk, csc, d, wrow, gram, 9)
    l = 4
    Wp, colmax_l = t("Wp", (d, l)), t("colmax_l", (l, 4))
    s("csr_panel/colmax", be.csr_panel_chunk, blk, d, Wp, colmax=colmax_l, row_offset=3)
    s("csr_panel/out", be.csr_panel_chunk, blk64, d, Wp, out=t("panel", (n, 6), f32)[:, :l])
    s("csr_panel/rows0", be.csr_panel_chunk, blk0, d, Wp, out=t("panel0", (0, l)))
    P, cout = t("P", (n, l)), t("cout", (d, l))
    s("csc_panel/first", be.csc_panel_chunk, csc, d, P, cout, first=True)
    s("csc_panel/next", be.csc_panel_chunk, csc, d, P, cout)
    s("sparse_pack/new", be.sparse_pack_centers, C64)
    spack = t("spack", d * k + k)
    s("sparse_pack/out", be.sparse_pack_centers, C64, out=spack)
    dist_sum, mind = t("dist_sum", 1), t("mind", n)
    s("csr_assign/mode0_acc", be.csr_assign_chunk, blk, d, spack, k, labels, mind, True, dist_sum, counts, first=True,
      loop_state=loop)
    s("csr_assign/mode0", be.csr_assign_chunk, blk64, d, spack, k, labels, mind, False)
    s("csr_assign/mode1", be.csr_assign_chunk, blk, d, spack, k, out=out_nk[:, 1:4], mode=1)
    s("csr_assign/mode2", be.csr_assign_chunk, blk, d, spack, k, out=t("dist64", (n, k)), mode=2)
    s("csr_assign/rows0", be.csr_assign_chunk, blk0, d, spack, k, out=out_nk[:0], mode=1)
    sumsT = t("sumsT", (d, k))
    s("csc_label_sums/first", be.csc_label_sums_chunk, csc, d, labels, k, sumsT, first=True, loop_state=loop)
    s("csc_label_sums/next", be.csc_label_sums_chunk, csc, d, labels, k, sumsT)
    spack2 = t("spack2", d * k + k)
    s("sparse_finalize_step", be.sparse_finalize_step, red, spack, spack2, state, k, d)
    s("sparse_minibatch_step", be.sparse_minibatch_step, red, spack, w_in, spack2, w_out, k, d)
    s("csr_kernel_colsum/first", be.csr_kernel_colsum, blk, d, spack, l, 0.125, colsum, first=True)
    s("csr_kernel_colsum/next", be.csr_kernel_colsum, blk64, d, spack, l, 0.125, colsum)
    Wk, emb = t("Wk", (l, 2)), t("emb", (n, 4), f32)
    s("csr_nystrom_embed", be.csr_nystrom_embed, blk, d, spack, l, 0.125, Wk, emb[:, :2])
    s("csr_nystrom_embed/rows0", be.csr_nystrom_embed, blk0, d, spack, l, 0.125, Wk, emb[:0, :2])
    s("nystrom_embed", be.nystrom_embed, x, pack, l, 0.5, Wk, emb[:, :2])
    s("nystrom_embed/rows0", be.nystrom_embed, x0, pack, l, 0.5, Wk, emb[:0, :2])
    Pn = 2
    prm = _lib.SgdParams(loss=1, penalty=2, learning_rate=3, fit_intercept=1, epsilon=0.1, alpha=1e-4, l1_ratio=0.15,
                         eta0=0.01, optimal_init=2.5, t0=1.0, intercept_decay=0.01, average=0.0)
    order, ys, eta, cw = t("order", (Pn, n), i32), t("ys", (Pn, n)), t("eta", n), t("cw", (Pn, 2))
    sw_, aw, q, st = t("sgd_w", (Pn, d)), t("sgd_aw", (Pn, d)), t("sgd_q", (Pn, d)), t("sgd_st", (Pn, 4))
    s("sgd_block", be.sgd_block, x, order, ys, wrow, None, cw, prm, sw_, aw, q, st)
    s("sgd_csr_block", be.sgd_csr_block, blk, d, order, ys, None, eta, cw, prm, sw_, aw, q, st)
    acc, minmax = t("acc", (5, d)), t("minmax", (2, d))
    s("colstats/first", be.colstats_chunk, x, shift, acc, minmax, first=True)
    s("colstats/next", be.colstats_chunk, xpad, None, acc, minmax)
    T = 2
    s("radix_state_new", be.radix_state_new, d, T)
    rstate, rhist = t("rstate", 256, u8), t("rhist", (d, T, 256))
    s("radix_hist/first", be.radix_hist_chunk, x, rstate, T, 0, rhist, first=True)
    s("radix_hist/next", be.radix_hist_chunk, x, rstate, T, 1, rhist)
    s("radix_select_step", be.radix_select_step, rhist, rstate, d, T, 1, f32, [0.25, 0.75])
    n_q = 3
    s("quantile_state_new", be.quantile_state_new, d, n_q)
    qstate, qhist = t("qstate", 512, u8), t("qhist", (d, 2 * n_q, 256))
    s("quantile_hist/first", be.quantile_hist_chunk, x, qstate, n_q, 0, qhist, first=True)
    s("quantile_hist/next", be.quantile_hist_chunk, x64, qstate, n_q, 2, qhist)
    s("quantile_select_step", be.quantile_select_step, qhist, qstate, d, n_q, 2, f64, t("qf", n_q))
    qT, ref, qout = t("qT", (d, n_q)), t("ref", n_q), t("qout", (n, 7))
    s("quantile_transform", be.quantile_transform_chunk, x, qT, ref, True, 1, -5.0, 5.0, qout[:, :d])
    s("quantile_transform/rows0", be.quantile_transform_chunk, x0, qT, ref, False, 0, 0.0, 1.0, qout[:0, :d])
    iacc = t("iacc", (4, d))
    s("impute_stats/first", be.impute_stats_chunk, x, True, 0.0, shift, iacc, first=True)
    s("impute_stats/next", be.impute_stats_chunk, x64, False, -1.0, None, iacc)
    s("quantile_hist_masked/first", be.quantile_hist_masked_chunk, x, -1.0, qstate, n_q, 0, qhist, first=True)
    s("quantile_hist_masked/next", be.quantile_hist_masked_chunk, x, 2.0, qstate, n_q, 1, qhist)
    g, total = 2, 16
    keys, kcounts, off = t("keys", total, i64), t("kcounts", total, i64), t("off", g + 1, i64)
    s("mode_count/first", be.mode_count_chunk, x[:, :g], True, 0.0, keys, kcounts, off, total, first=True)
    s("mode_count/next", be.mode_count_chunk, x64[:, 1:3], False, -1.0, keys, kcounts, off, total)
    s("mode_best", be.mode_best, keys, kcounts, off, g, total)
    entries = t("entries", (total, 4))
    s("mode_compact", be.mode_compact, keys, kcounts, off, g, entries)
    s("mode_merge", be.mode_merge, entries, keys, kcounts, off, g, total)
    stats, cols, iout = t("stats", d), t("cols", d, i32), t("iout", (n, 8), f32)
    s("impute", be.impute_chunk, x, True, 0.0, stats, cols, 4, 1, 2, False, iout[:, :6], invalid=t("invalid", 2))
    s("impute/inverse", be.impute_chunk, x64, False, -1.0, stats, cols, 4, 1, 0, True, t("iout64", (n, d)))
    s("impute/rows0", be.impute_chunk, x0, False, -1.0, stats, cols, 4, 1, 0, False, iout[:0, :6])
    dstate = t("dstate", (2, g), i64)
    s("distinct/first", be.distinct_chunk, xi, keys, kcounts, off, total, dstate, first=True)
    s("distinct/next", be.distinct_chunk, x[:, :g], keys, kcounts, off, total, dstate)
    s("distinct/full", be.distinct_chunk, x[:, :g], keys, kcounts, off, total, dstate, full_probe=True)
    cat_keys, cat_off, unknown = t("cat_keys", 8, i64), t("cat_off", 3, i64), t("unknown", 1 + 2 + 2 * 8, i64)
    codes = t("codes", (n, 4), i32)
    s("encode/codes", be.encode_chunk, xi, cat_keys, cat_off, 7, _lib.ENCODE_CODES, codes[:, :2], unknown)
    s("encode/codes_rows0", be.encode_chunk, xi[:0], cat_keys, cat_off, 7, _lib.ENCODE_CODES, codes[:0, :2], unknown)
    s("encode/dense", be.encode_chunk, xi, cat_keys, cat_off, 7, _lib.ENCODE_DENSE, t("onehot", (n, 7), f32), unknown)
    s("encode/csr", be.encode_chunk, x[:, :2], cat_keys, cat_off, 7, _lib.ENCODE_CSR, t("csr_data", n * 2), unknown,
      indices=t("csr_idx", n * 2, i64))
    cat_vals = t("cat_vals", 8, i64)
    s("decode", be.decode_chunk, codes[:, 1:3], cat_vals, cat_off, t("dec", (n, 2), i64), unknown)
    s("decode/rows0", be.decode_chunk, codes[:0, :2], t("cat_vals32", 8, f32), cat_off, t("dec0", (0, 2), f32),
      unknown)
    buf, doc_off = t("buf", 24, u8), t("doc_off", 3, i64)
    tok_start, tok_off, pair_off, totals = t("tok_start", 9, i64), t("tok_off", 3, i64), t("pair_off", 3, i64), \
        t("totals", 3, i64)
    s("text_tokens", be.text_tokens_chunk, buf, doc_off, 1, 2, tok_start, tok_off, pair_off, totals)
    tkeys, indptr, scale = t("tkeys", 7, i32), t("indptr", 3, i64), t("scale", 2)
    s("text_hash/none", be.text_hash_chunk, buf, tok_start, tok_off, pair_off, 5, 7, 1, 2, True, 1 << 20, True, False,
      None, f32, tkeys, indptr, scale, totals)
    s("text_hash/l2", be.text_hash_chunk, buf, tok_start, tok_off, pair_off, 5, 7, 1, 1, False, 64, False, True, "l2",
      f64, tkeys, indptr, scale, totals)
    s("text_write", be.text_write_chunk, tkeys, pair_off, indptr, scale, True, t("tidx", 7, i64), t("tdata", 7, f32))
    a, b, aout = t("a", d), t("b", d), t("aout", (n, 8), f32)
    s("affine", be.affine_chunk, x, a, b, 1, 1, aout[:, :d])
    s("affine/none", be.affine_chunk, x64, None, b, 0, 2, t("aout64", (n, d)))
    s("affine/rows0", be.affine_chunk, x0, a, None, 2, 0, aout[:0, :d])
    s("split_indices", be.split_indices_chunk, 0xDEADBEEF, 100, 10, 20, 1000)
    idx = t("idx", 4, i64)
    s("gather/rows", be.gather_rows_chunk, xpad, idx, idx_offset=2)
    s("gather/1d", be.gather_rows_chunk, labels, idx)
    s("gather/one_row", be.gather_rows_chunk, x64[:1], idx, idx_offset=5)
    s("gather/none", be.gather_rows_chunk, x, idx[:0])
    macc, mw = t("macc", (4, 2)), t("mw", n)
    s("metric/eq", be.metric_chunk, t("ma", n, i64), t("mb", n, i64), _lib.METRIC_EQ, macc, first=True)
    s("metric/err", be.metric_chunk, t("ea", (n, 2)), t("eb", (n, 2), f32), _lib.METRIC_ERR, macc, w=mw,
      shift=t("mshift", 2))
    s("metric/logloss", be.metric_chunk, t("la", n, i32), t("lb", (n, 3)), _lib.METRIC_LOGLOSS, macc, eps=1e-15,
      first=True)
    s("metric/bool", be.metric_chunk, t("ba", n, torch.bool), t("bb", n, u8), _lib.METRIC_EQ, macc)
    s("finalize", be.finalize, sums, counts, C64, c_out, t("fshift", 1))


def _drive_datasets(rec):
    """The device paths of the dataset generators and the SGD row orders."""
    centers = np.array([[0.0, 1.0, 2.0], [3.0, 4.0, 5.0]])
    rec.step("make_blobs", datasets.make_blobs, n_samples=7, n_features=3, centers=centers, cluster_std=[1.0, 2.0],
             chunks=4, device="cpu", dtype=np.float32)
    info = np.array([[1.0, 0.5], [0.0, -0.25]])
    rec.step("generate/normal", datasets._generate, [3, 2], 4, None, datasets._NORMAL, info, 123, "cpu", n_targets=2,
             bias=0.5, noise=1.5)
    rec.step("generate/poisson", datasets._generate, [5], 4, np.float32, datasets._POISSON, info, 77, "cpu")
    real_empty = torch.empty

    def empty(*args, **kw):            # _normal_panel takes its device path only for a CUDA device
        kw["device"] = "cpu"
        return real_empty(*args, **kw)

    torch.empty = empty
    try:
        rec.step("normal_panel", datasets._normal_panel, 99, 5, 3, torch.device("cuda", 0))
        rec.step("normal_panel/rows0", datasets._normal_panel, 99, 0, 3, torch.device("cuda", 0))
    finally:
        torch.empty = real_empty
    rec.step("sgd_orders", _sgd._PartialSGDMixin._orders, types.SimpleNamespace(shuffle=True), 5, [3, 1 << 40])


def _install(monkeypatch):
    """A GPU as far as the backend can tell, and the fake library in place of the real one."""
    lib = _FakeLib()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "device", _Device)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: _Stream())
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(_lib, "_lib", lib)
    monkeypatch.delenv("BKM_FLAGS", raising=False)
    return lib


def _record(monkeypatch):
    lib = _install(monkeypatch)
    be = engine.CudaBackend(device="cpu", flags=_lib.FLAG_NO_RECHECK)
    rec = _Recorder(lib, be)
    _drive(rec, be)
    _drive_datasets(rec)
    return rec.log


def _dump(log):
    return "[\n" + ",\n".join(json.dumps(e) for e in log) + "\n]\n"


def test_every_entry_point_is_driven(monkeypatch):
    reached = {e[1] for e in _record(monkeypatch)}
    expected = {n for n in _lib.SIGNATURES if not n.startswith(NOT_DRIVEN)}
    assert expected - reached == set()


def test_failed_call_raises_with_its_name(monkeypatch):
    """A non-zero status raises RuntimeError naming the entry point and carrying the library's message."""
    lib = _install(monkeypatch)
    monkeypatch.setattr(lib, "bkm_gram_chunk", lambda *args: -3)
    monkeypatch.setattr(lib, "bkm_error_string", lambda rc: b"shape not supported by any kernel")
    be = engine.CudaBackend(device="cpu")
    x, v, g = torch.zeros((4, 3)), torch.zeros(3, dtype=torch.float64), torch.zeros((3, 3), dtype=torch.float64)
    with pytest.raises(RuntimeError, match=r"bkm_gram_chunk failed: shape not supported by any kernel \(code -3\)"):
        be.gram_chunk(x, None, v, g)


def test_calls_match_golden(monkeypatch):
    got = json.loads(_dump(_record(monkeypatch)))
    with open(GOLDEN) as f:
        want = json.load(f)
    for g, w in zip(got, want):
        assert g == w, "\n got  %s\n want %s" % (json.dumps(g), json.dumps(w))
    assert len(got) == len(want)


if __name__ == "__main__":
    if sys.argv[1:] != ["--record"]:
        sys.exit("usage: python tests/test_backend_calls_host.py --record")
    with pytest.MonkeyPatch.context() as mp:
        text = _dump(_record(mp))
    with open(GOLDEN, "w") as f:
        f.write(text)
    print("wrote %s" % GOLDEN)
