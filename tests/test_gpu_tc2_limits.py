"""The large-shape tensor path (bf16 rows, d <= 128, k <= 4096) at its limits, on data whose every distance is exact
(run with -m gpu).  The cases and the data come from tests/tc2_cases.py, which the CPU test test_tc2_cases_host.py
pins against the library's layout query at 132 and 114 SMs; here they run at the device's own SM count.

Every case designs its rows so that the deferred set is known in advance: near-ties of 2^-18 in either order and exact
ties at the MMA fragment neighbours of every slice, across every slice border and between slice 0 and the last
column; rows that win in one slice while a losing slice holds a near-tie of its own (which must NOT be deferred);
duplicate centres at every reduction level of the float64 re-check; and far rows, decided on the tensor path, labelled
by every column in the slice-count cases (the single column of the last slice at k = 3841 included).  Outputs are
poisoned before each call (labels -1, distances NaN, the workspace's slice records, and for the call without labels
its label buffer), and each call must give:

* labels equal to the float64 arg-min (lowest index on exact ties), and exactly the designed number of deferred rows;
* counts exact, sums bit-identical to the order-exact row-pass reference (msum_ref);
* squared and plain distances bit-equal to the float64 direct form rounded to fp32, inertia and the distance sum
  bit-equal to the restated fold;
* the same from assign_chunk (labels only; labels + distances), from lloyd_chunk without labels (the workspace label
  buffer, poisoned too), and from a second call on the warm workspace.

The labels-only call runs first and its labels are checked before any call that runs the row passes: those index
the centres and the cluster sums by label, so a label out of [0, k) must stop the test there.

test_fit_matches_float64_lloyd runs KMeans.fit itself at k ~ 2000 and 4096 on ragged bf16 chunks for 3 iterations
(the pack rebuilt and the balance table carried between iterations) against a float64 Lloyd on the device.
"""
import numpy as np
import pytest

import msum_ref as mr
import tc2_cases as tc
from _util import sm_count

pytestmark = pytest.mark.gpu

CASE_IDS = [c["id"] for c in tc.cases(132)]


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


@pytest.fixture(scope="module")
def sms(be):
    return sm_count(be.lib, be.device.index or 0)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def _assert_bits(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    bad = _bits(got) != _bits(want)
    assert not bad.any(), "%s: %d values differ, first at %s (got %r, want %r)" % (
        what, int(bad.sum()), np.argwhere(bad)[0].tolist(), got[bad][0], want[bad][0])


def _want(X, C, lab, k, sms):
    """Expected (sums, counts, min_d2, dist, inertia, dist_sum) of the designed rows."""
    X32 = X.astype(np.float32)
    sums = mr.reduce_partials(mr.rowpass_partials(X32, lab, k, sms))
    d2 = ((X - C[lab]) ** 2).sum(1)
    dist = np.sqrt(d2)
    return dict(sums=sums, counts=np.bincount(lab, minlength=k), md=d2.astype(np.float32),
                dist=dist.astype(np.float32), inertia=tc.dist_sum_ref(d2, sms), dist_sum=tc.dist_sum_ref(dist, sms))


def _poison_records(be, n, d, k, sms):
    """Fill the workspace's per-(slice, row) records with 0xff bytes (NaN minima, label -1): a record the assign kernel
    fails to write must not pass for one a previous call left behind."""
    import torch

    S = tc.tc2_geom(k, d)["S"]
    if S > 1:
        W = tc.ws_layout(n, d, k, sms)
        be._workspace(n, d, k, torch.bfloat16)[W["rec"]:W["rec"] + S * n * 16].fill_(255)


def _labels_first(be, x, pack, k, sms, lab, where):
    """The labels-only call (no row pass), its labels checked at once: {labels, deferred}."""
    import torch

    n, d = x.shape
    labels = be.empty((n,), torch.int32).fill_(-1)
    _poison_records(be, n, d, k, sms)
    be.assign_chunk(x, pack, k, labels, None, True, None)
    torch.cuda.synchronize()
    got = labels.cpu().numpy()
    bad = np.nonzero(got != lab)[0]
    assert len(bad) == 0, "%s assign: %d labels differ, first row %d: %d for %d" % (
        where, len(bad), bad[0], got[bad[0]], lab[bad[0]])
    return dict(labels=got, deferred=be.deferred_rows(n, d, k, torch.bfloat16))


def _outputs(be, x, pack, k, sms, n, d, lab, where):
    """Every call form on x, outputs poisoned first: a dict of numpy results per call."""
    import torch

    out = {"assign": _labels_first(be, x, pack, k, sms, lab, where)}
    labels = be.empty((n,), torch.int32)
    md = be.empty((n,), torch.float32)

    def lloyd(tag, with_labels=True):
        sums, counts, inertia = be.zeros((k * d,), torch.float64), be.zeros((k,), torch.int64), be.zeros((1,), torch.float64)
        labels.fill_(-1)
        md.fill_(float("nan"))
        _poison_records(be, n, d, k, sms)
        if not with_labels:
            W = tc.ws_layout(n, d, k, sms)
            be._workspace(n, d, k, torch.bfloat16)[W["lab"]:W["lab"] + 4 * n].view(torch.int32).fill_(-1)
        be.lloyd_chunk(x, pack, k, labels if with_labels else None, md if with_labels else None, sums, counts,
                       inertia if with_labels else None)
        torch.cuda.synchronize()
        out[tag] = dict(sums=sums.cpu().numpy().reshape(k, d), counts=counts.cpu().numpy(),
                        deferred=be.deferred_rows(n, d, k, torch.bfloat16))
        if with_labels:
            out[tag].update(labels=labels.cpu().numpy(), md=md.cpu().numpy(), inertia=float(inertia[0]))

    lloyd("lloyd")
    labels.fill_(-1)
    md.fill_(float("nan"))
    ds = be.zeros((1,), torch.float64)
    _poison_records(be, n, d, k, sms)
    be.assign_chunk(x, pack, k, labels, md, False, ds)
    torch.cuda.synchronize()
    out["assign-dist"] = dict(labels=labels.cpu().numpy(), dist=md.cpu().numpy(), dist_sum=float(ds[0]),
                              deferred=be.deferred_rows(n, d, k, torch.bfloat16))
    lloyd("lloyd-nolabels", with_labels=False)
    lloyd("lloyd-warm")
    return out


def _check(out, lab, n_def, want, where):
    for tag, o in out.items():
        w = "%s %s" % (where, tag)
        assert o["deferred"] == n_def, "%s: %d deferred rows, designed %d" % (w, o["deferred"], n_def)
        if "labels" in o:
            bad = np.nonzero(o["labels"] != lab)[0]
            assert len(bad) == 0, "%s: %d labels differ, first row %d: %d for %d" % (
                w, len(bad), bad[0], o["labels"][bad[0]], lab[bad[0]])
        if "counts" in o:
            np.testing.assert_array_equal(o["counts"], want["counts"], err_msg=w)
            _assert_bits(o["sums"], want["sums"], w + " sums")
        if "md" in o:
            _assert_bits(o["md"], want["md"], w + " min_d2")
            assert o["inertia"] == want["inertia"], (w, o["inertia"], want["inertia"])
        if "dist" in o:
            _assert_bits(o["dist"], want["dist"], w + " distances")
            assert o["dist_sum"] == want["dist_sum"], (w, o["dist_sum"], want["dist_sum"])


def _device(be, X, C):
    import torch

    x = be.to_device(torch.from_numpy(X.astype(np.float32)), torch.bfloat16)
    pack = be.pack_centers(torch.as_tensor(C).to(be.device), torch.bfloat16)
    return x, pack


@pytest.mark.parametrize("cid", CASE_IDS)
def test_case(be, sms, cid):
    import torch

    c = {c["id"]: c for c in tc.cases(sms)}[cid]
    d, k, n = c["d"], c["k"], c["n"]
    assert be.kernel_family(d, k, torch.bfloat16) == 3
    X, C, lab, deferred, kinds = tc.design(d, k, n, seed=n + 7 * k + d, n_defer=c["n_defer"])
    n_def = int(deferred.sum())
    if c["n_defer"] is not None:
        assert n_def == c["n_defer"]
    x, pack = _device(be, X, C)
    out = _outputs(be, x, pack, k, sms, n, d, lab, cid)
    _check(out, lab, n_def, _want(X, C, lab, k, sms), cid)


POISON_D = (1, 9, 33, 65, 100, 127)


@pytest.mark.parametrize("d", POISON_D)
def test_poisoned_pitch(be, sms, d):
    """Rows in an (n, pitch) buffer whose padding holds NaN, then +-3e38: every output bit-identical to the expected
    (and so to the zero-padded run)."""
    import torch

    k = min(100, 2 ** max(1, d - 2))
    n = 64 * 9 + 17
    X, C, lab, deferred, kinds = tc.design(d, k, n, seed=d)
    want = _want(X, C, lab, k, sms)
    pitch = (d + 7) // 8 * 8 + 8
    pack = be.pack_centers(torch.as_tensor(C).to(be.device), torch.bfloat16)
    for fill in ("nan", "big"):
        buf = torch.empty((n, pitch), dtype=torch.bfloat16, device=be.device)
        if fill == "nan":
            buf.fill_(float("nan"))
        else:
            buf[:, 0::2] = 3e38
            buf[:, 1::2] = -3e38
        buf[:, :d] = torch.from_numpy(X.astype(np.float32)).to(be.device, torch.bfloat16)
        x = buf[:, :d]
        assert x.stride(0) == pitch
        where = "d=%d pitch=%d padding %s" % (d, pitch, fill)
        out = _outputs(be, x, pack, k, sms, n, d, lab, where)
        _check(out, lab, int(deferred.sum()), want, where)


BAL = [(128, 2048), (128, 4096)] + [(128, kt + o) for kt in tc.ds_transitions(128) for o in (-1, 0)]


@pytest.mark.parametrize("d,k", BAL, ids=["d%d-k%d" % s for s in BAL])
def test_balance_table_states(be, sms, d, k):
    """The row pass's cluster -> warp balance table absent, present (left by the previous call) and stale (same
    header, warps dealt at random): the sums stay bit-identical to the order-exact reference."""
    import torch

    n = 3 * 4096 + 77
    X, C, lab, deferred, kinds = tc.design(d, k, n, seed=k)
    want = _want(X, C, lab, k, sms)
    x, pack = _device(be, X, C)
    first = _labels_first(be, x, pack, k, sms, lab, "d=%d k=%d" % (d, k))
    assert first["deferred"] == int(deferred.sum()), (first["deferred"], int(deferred.sum()))
    ds = tc.tc2_geom(k, d)["DS"]
    rng = np.random.RandomState(k)
    for state in ("absent", "present", "stale"):
        ws = be._workspace(n, d, k, torch.bfloat16)
        if state == "absent":
            ws[:8192].zero_()
        hdr = ws[:16].view(torch.int32).cpu().numpy()
        if state == "present":
            assert hdr[0] == 0x62616c31 and hdr[1] == k and hdr[2] == ds, hdr
        if state == "stale":
            ws[16:16 + k] = torch.from_numpy(rng.randint(0, 16, k).astype(np.uint8)).to(be.device)
        sums, counts = be.zeros((k * d,), torch.float64), be.zeros((k,), torch.int64)
        labels = be.empty((n,), torch.int32).fill_(-1)
        be.lloyd_chunk(x, pack, k, labels, None, sums, counts, None)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(labels.cpu().numpy(), lab)
        np.testing.assert_array_equal(counts.cpu().numpy(), want["counts"])
        _assert_bits(sums.cpu().numpy().reshape(k, d), want["sums"], "balance table " + state)


def _lloyd64(X64, C, iters):
    """float64 Lloyd on the device: ``iters`` (E-step, centre update) rounds from C, an empty cluster's centre set to 0
    (bkm_finalize_step).  Returns the centres after each round."""
    import torch

    out = []
    k = C.shape[0]
    for _ in range(iters):
        lab = _argmin64(X64, C)[0]
        sums = torch.zeros_like(C).index_add_(0, lab, X64)
        cnt = torch.bincount(lab, minlength=k).to(C.dtype)
        C = sums / cnt.clamp(min=1.0)[:, None]
        out.append(C)
    return out


def _argmin64(X64, C):
    """(labels, top-2 margin) of the float64 E-step, ||c||^2 - 2 x.c, in row blocks."""
    import torch

    cn = (C * C).sum(1)
    lab = torch.empty(X64.shape[0], dtype=torch.int64, device=X64.device)
    margin = torch.empty(X64.shape[0], dtype=torch.float64, device=X64.device)
    for s in range(0, X64.shape[0], 8192):
        e = cn[None, :] - 2.0 * X64[s:s + 8192] @ C.T
        top = torch.topk(e, 2, dim=1, largest=False)
        lab[s:s + 8192] = top.indices[:, 0]
        margin[s:s + 8192] = top.values[:, 1] - top.values[:, 0]
    return lab, margin


@pytest.mark.parametrize("k", [1999, 4096])
def test_fit_matches_float64_lloyd(be, k):
    """KMeans.fit on ragged bf16 chunks, 3 iterations from k distinct rows, against the float64 Lloyd restatement with
    the same init: the centres within the fp32 partial-sum tolerance, labels_ (a re-label against the final centres:
    they still move) equal to the float64 arg-min except on float64 near-ties."""
    import torch
    from dask_ml_b200.chunked import ChunkedArray
    from dask_ml_b200.cluster import KMeans

    n, d, iters = 20 * k + 123, 128, 3
    g = torch.Generator(device=be.device).manual_seed(k)
    cent = torch.empty((k // 4, d), device=be.device).uniform_(-10, 10, generator=g)
    X = (cent[torch.randint(0, k // 4, (n,), device=be.device, generator=g)] +
         torch.randn((n, d), device=be.device, generator=g)).to(torch.bfloat16)
    assert be.kernel_family(d, k, torch.bfloat16) == 3
    init = X[torch.randperm(n, device=be.device, generator=g)[:k]].double()
    assert torch.unique(init, dim=0).shape[0] == k
    cuts = [0, n // 3, n // 3 + 1, (3 * n) // 4, n]
    parts = ChunkedArray([X[a:b] for a, b in zip(cuts, cuts[1:])])
    km = KMeans(n_clusters=k, init=init.float().cpu().numpy(), max_iter=iters, tol=0.0).fit(parts)
    X64 = X.double()
    Cs = _lloyd64(X64, init, iters)
    C_ref = Cs[-1]
    assert float(((Cs[-1] - Cs[-2]) ** 2).sum()) > 1e-3          # still moving: labels_ is the re-label
    assert km.n_iter_ == iters
    got_C = torch.as_tensor(km.cluster_centers_).to(be.device).double()
    tol = 4e-6 * float(C_ref.abs().max())
    err = float((got_C - C_ref).abs().max())
    assert err <= tol, (err, tol)
    want, margin = _argmin64(X64, C_ref)
    got = torch.as_tensor(np.asarray(km.labels_.compute())).to(be.device).long()
    bad = got != want
    scale = (X64 ** 2).sum(1) + (C_ref ** 2).sum(1).max()
    assert int(bad.sum()) == 0 or bool((margin[bad] <= 1e-9 * scale[bad]).all()), int(bad.sum())
    assert int(bad.sum()) <= 3
