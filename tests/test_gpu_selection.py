"""The exact order-statistic passes on the device, on the adversarial columns of selection_cases.py.

The round loop of order_statistics is driven by hand through CudaBackend and the numpy restatement of the passes
(QTOracleBackend) side by side on the same chunks: after every hist pass the device histogram, and after every
select step the device state (head nvalid / R / L, every distinct rank's record, the live list), must equal the
restatement's byte for byte, so a failure names the case, the split, the round and the column.  Every plan entry runs
whole; the n_q = 57 and 1000 entries also run in ragged chunks and in chunks that end at the target ranks of column 0.
Then
the public results on the same columns: quantiles_ and the uniform transform, the radix percentiles, SimpleImputer's
median and most_frequent; and the state's stability over two calls and over column-group splits."""
import os
import sys
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import selection_cases as sc  # noqa: E402
from test_impute_host import ImputeOracleBackend  # noqa: E402
from test_quantile_host import _state_views, transform_restated  # noqa: E402
from test_selection_host import QSETS, check_order_statistics, sk_imputer  # noqa: E402

RAGGED = (1, 255, 1000, 7, 3333, 64)


def _backend():
    from dask_ml_b200.cluster import k_means as km

    return km._get_backend()


def _id(e):
    name, dt, d, nq, missing = e
    return "%s-%s-d%d-nq%d%s" % (name, dt, d, nq, "" if missing is None else "-miss%g" % missing)


def split_rows(case, nq, missing, kind):
    """(row order, chunk sizes): whole; ragged; or the rows sorted by column 0 (valid values ascending, then the rest)
    with a chunk boundary at each of its target ranks r and r + 1."""
    n = case.n
    if kind == "whole":
        return np.arange(n), [n]
    if kind == "ragged":
        sizes, i = [], 0
        while sum(sizes) < n:
            sizes.append(min(RAGGED[i % len(RAGGED)], n - sum(sizes)))
            i += 1
        return np.arange(n), sizes
    v = case.values()[:, 0]
    ok = ~np.isnan(v) if missing is None else ~np.isnan(v) & (v != missing)
    key = sc.key_of(case.dt, case.bits[:, 0]).astype(np.float64)
    order = np.lexsort((key, ~ok))
    m = int(ok.sum())
    r = sc.target_ranks(m, sc.references(nq))
    cuts = np.unique(np.concatenate([[0, n], r, r + 1]))
    cuts = cuts[(cuts >= 0) & (cuts <= n)]
    return order, list(np.diff(cuts))


def hist_pass(be, x, state, nq, rnd, hist, first, missing):
    if missing is None:
        be.quantile_hist_chunk(x, state, nq, rnd, hist, first=first)
    else:
        be.quantile_hist_masked_chunk(x, missing, state, nq, rnd, hist, first=first)


def first_difference(got, want, what):
    at = tuple(int(i) for i in np.argwhere(got != want)[0])
    return "%s differs at %s: device %r, restatement %r" % (what, at, got[at].item(), want[at].item())


def compare_state(sd, so, d, nq, where):
    hd, rd, ld = _state_views(sd, d, nq)
    ho, ro, lo = _state_views(so, d, nq)
    for f in ("nvalid", "R", "L"):
        assert np.array_equal(hd[f], ho[f]), "%s: %s" % (where, first_difference(hd[f], ho[f], "head " + f))
    for j in range(d):
        R, L = int(ho["R"][j]), int(ho["L"][j])
        a, b = rd[j, :R], ro[j, :R]
        if a.tobytes() != b.tobytes():
            for f in ("key", "rank", "nvalid", "slot", "pad"):
                assert np.array_equal(a[f], b[f]), "%s column %d: %s" % (where, j, first_difference(a[f], b[f], f))
        assert np.array_equal(ld[j, :L], lo[j, :L]), "%s column %d: %s" % (where, j, first_difference(
            ld[j, :L], lo[j, :L], "live"))


def drive(be, chunks, d, nq, dt, missing, state, qf, check=None):
    """The round loop of order_statistics over ``chunks`` into ``state``; ``check(rnd, hist)`` after each round's hist
    passes."""
    rounds = sc.BITS[dt] // 8
    hist = be.zeros((d * min(2 * nq, 256 ** (rounds - 1)) * 256,), torch.float64)
    for rnd in range(rounds):
        h = hist[: d * min(2 * nq, 256 ** rnd) * 256]
        for i, x in enumerate(chunks):
            hist_pass(be, x, state, nq, rnd, h, i == 0, missing)
        if check is not None:
            check(rnd, h, "hist")
        be.quantile_select_step(h, state, d, nq, rnd, sc.TORCH[dt], qf)
        if check is not None:
            check(rnd, state, "state")
    return state


def oracle_rounds(case, nq, missing):
    """The restatement's histogram and state after each round, over all rows at once (the counts of a round are sums
    over rows, so they do not depend on the chunking): [(hist (d, cap, 256), state)]."""
    orc, d, dt = ImputeOracleBackend(), case.d, case.dt
    qf = torch.as_tensor(sc.references(nq))
    state = orc.quantile_state_new(d, nq)
    out = []
    for rnd in range(sc.BITS[dt] // 8):
        h = torch.zeros(d * min(2 * nq, 256 ** rnd) * 256, dtype=torch.float64)
        hist_pass(orc, case.tensor(), state, nq, rnd, h, True, missing)
        want = h.view(d, -1, 256).numpy().copy()
        orc.quantile_select_step(h, state, d, nq, rnd, sc.TORCH[dt], qf)
        out.append((want, state.clone()))
    return out


def replay(entry, kinds):
    """The device's round loop on the entry's case, split as each of ``kinds`` says, against the restatement after
    every hist pass and every select step."""
    name, dt, d, nq, missing = entry
    case = sc.make(name, dt, d, nq)
    want = oracle_rounds(case, nq, missing)
    be = _backend()
    qf = torch.as_tensor(sc.references(nq)).cuda()
    for kind in kinds:
        order, sizes = split_rows(case, nq, missing, kind)
        t = case.tensor()[torch.as_tensor(order)].cuda()
        offs = np.concatenate([[0], np.cumsum(sizes)])
        where = "%s %s" % (_id(entry), kind)

        def check(rnd, dev, what):
            if what == "hist":
                got = dev.cpu().view(d, -1, 256).numpy()
                assert np.array_equal(got, want[rnd][0]), "%s round %d: %s" % (
                    where, rnd, first_difference(got, want[rnd][0], "hist"))
            else:
                compare_state(dev.cpu(), want[rnd][1], d, nq, "%s round %d" % (where, rnd))

        drive(be, [t[a:b] for a, b in zip(offs[:-1], offs[1:])], d, nq, dt, missing, be.quantile_state_new(d, nq),
              qf, check)


PLAN = sc.plan()


@pytest.mark.parametrize("entry", PLAN, ids=_id)
def test_replay(entry):
    """Whole; and for n_q 57 and 1000 also in ragged chunks and in chunks that end at column 0's target ranks."""
    replay(entry, ("whole", "ragged", "at_ranks") if entry[3] in (57, 1000) else ("whole",))


# ------------------------------------------------ public results ------------------------------------------------
def chunked(case, rows):
    from dask_ml_b200 import ChunkedArray

    t = case.tensor()
    return ChunkedArray([t[i:i + rows].cuda() for i in range(0, case.n, rows)])


@pytest.mark.parametrize("dt", sc.DTYPES)
@pytest.mark.parametrize("name", ["full_range", "one_prefix", "carry", "zero_carry", "boundary"])
def test_quantile_transformer(name, dt):
    """quantiles_ equal np.percentile and the uniform transform equals the restatement bit for bit."""
    from dask_ml_b200.preprocessing import QuantileTransformer

    for nq in (57, 1000):
        case = sc.make(name, dt, sc.sector(dt) + 1, nq)
        v = case.values()
        qt = QuantileTransformer(n_quantiles=nq, subsample=10 ** 6).fit(chunked(case, 1777))
        with np.errstate(all="ignore"):
            want = np.percentile(v, qt.references_ * 100, axis=0)
            np.testing.assert_array_equal(qt.quantiles_, want, err_msg="%r nq=%d" % (case, nq))
            got = qt.transform(chunked(case, 2500)).compute()
            np.testing.assert_array_equal(got, transform_restated(v, qt.quantiles_, qt.references_, False, "uniform"),
                                          err_msg="%r nq=%d transform" % (case, nq))


@pytest.mark.parametrize("dt", sc.DTYPES)
@pytest.mark.parametrize("name", ["full_range", "one_prefix", "carry", "zero_carry", "boundary", "specials"])
def test_radix_percentiles(name, dt):
    """percentiles (bkm_radix_*) equal np.nanpercentile of every NaN-free column, NaN where the column holds a NaN."""
    from dask_ml_b200.decomposition.pca import _device_data
    from dask_ml_b200.preprocessing.data import percentiles

    case = sc.make(name, dt, 3 * sc.sector(dt) + 1)
    X = _device_data(chunked(case, 2500), allow_nonfinite=True)
    v = case.values()
    for q in QSETS:
        got = percentiles(X, list(q))
        with np.errstate(all="ignore"), warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            want = np.stack([np.nanpercentile(v[:, j], q) for j in range(case.d)])
        want[np.isnan(v).any(0)] = np.nan
        np.testing.assert_array_equal(got, want, err_msg="%r q=%s" % (case, q))


@pytest.mark.parametrize("dt", sc.DTYPES)
@pytest.mark.parametrize("name,strategy", [("boundary", "median"), ("zero_carry", "median"), ("masked", "median"),
                                           ("masked_zero", "median"), ("specials", "median"),
                                           ("mode_ties", "most_frequent"), ("mode_many", "most_frequent"),
                                           ("masked_zero", "most_frequent"), ("zero_carry", "most_frequent")])
def test_imputer_statistics(name, strategy, dt):
    from dask_ml_b200.impute import SimpleImputer

    case = sc.make(name, dt, sc.sector(dt) + 1)
    fin = ~np.isinf(case.values()).any(0)                     # scikit-learn refuses inf
    case.bits = case.bits[:, fin]
    missing = np.nan if case.missing is None else case.missing
    got = SimpleImputer(strategy=strategy, missing_values=missing).fit(chunked(case, 1500))
    want = sk_imputer(case.values(), strategy, missing)
    np.testing.assert_array_equal(got.statistics_.astype(np.float64), want.statistics_.astype(np.float64),
                                  err_msg=repr(case))


@pytest.mark.parametrize("dt", sc.DTYPES)
def test_order_statistics_public(dt):
    """order_statistics on the device against np.sort, for the cases whose ranks sit on bin boundaries."""
    from dask_ml_b200.decomposition.pca import _device_data
    from dask_ml_b200.preprocessing.data import order_statistics

    for name, missing in (("boundary", None), ("specials", None), ("specials", 0.0), ("masked", 2.0)):
        case = sc.make(name, dt, 3 * sc.sector(dt) + 1, 57)
        lo, hi, m = order_statistics(_device_data(chunked(case, 999), allow_nonfinite=True), sc.references(57),
                                     missing=missing)
        check_order_statistics(case, 57, missing, lo, hi, m)


# ------------------------------------------------ stability ------------------------------------------------
@pytest.mark.parametrize("dt", sc.DTYPES)
@pytest.mark.parametrize("name,nq", [("full_range", 1000), ("boundary", 57), ("specials", 57), ("full_range", 10000)])
def test_state_stable_over_calls_and_column_groups(name, nq, dt):
    """Two calls write identical state, and so do column groups of 1, CS - 1 and CS + 2 columns read from strided
    views of the same chunks."""
    be = _backend()
    d = 3 * sc.sector(dt) + 1 if nq < 10000 else 5
    case = sc.make(name, dt, d, nq)
    t = case.tensor()
    chunks = [t[i:i + 3001].cuda() for i in range(0, case.n, 3001)]
    qf = torch.as_tensor(sc.references(nq)).cuda()
    a = drive(be, chunks, d, nq, dt, None, be.quantile_state_new(d, nq), qf).cpu()
    b = drive(be, chunks, d, nq, dt, None, be.quantile_state_new(d, nq), qf).cpu()
    assert torch.equal(a, b)
    stride = 16 + 80 * nq
    for g in (1, sc.sector(dt) - 1, sc.sector(dt) + 2):
        s = be.quantile_state_new(d, nq)
        for j0 in range(0, d, g):
            j1 = min(d, j0 + g)
            drive(be, [x[:, j0:j1] for x in chunks], j1 - j0, nq, dt, None, s[j0 * stride: j1 * stride], qf)
        assert torch.equal(s.cpu(), a), (name, dt, nq, g)
