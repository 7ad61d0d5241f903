"""The exact order-statistic passes without a GPU, on the adversarial columns of selection_cases.py: order_statistics,
QuantileTransformer.quantiles_, the radix percentiles of RobustScaler and SimpleImputer's median and most_frequent, each
run through the numpy restatements of the passes and checked against numpy / scikit-learn; and the coverage the cases
give the selection's live lists (how many live prefixes a round carries, and whether the hist pass stages them in
shared memory or searches them in global memory), which the GPU replay relies on."""
import os
import sys
import warnings

import numpy as np
import pytest
import sklearn.impute
import sklearn.preprocessing

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import selection_cases as sc  # noqa: E402
from test_impute_host import ImputeOracleBackend  # noqa: E402

STAGE_BYTES = 96 * 1024


def staged(dt, rnd, nq):
    """Whether a round-``rnd`` hist pass stages the live lists of its CTA's columns in shared memory: the rule of
    launch_qhist in csrc/bkm_quantile.cu, CS * cap * sizeof(key) <= 96 KiB with the key 8 bytes for fp64 and 4 for
    fp32 / bf16, cap = min(2 n_q, 256^rnd)."""
    cap = min(2 * nq, 256 ** rnd)
    return rnd > 0 and sc.sector(dt) * cap * (8 if dt == "f64" else 4) <= STAGE_BYTES


class RecordingBackend(ImputeOracleBackend):
    """The numpy passes, recording for every hist pass of round >= 1 the live list length L of each column it reads,
    and for every select step the distinct ranks R and the run layout of the live list it builds."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.hist_rounds = []             # (rnd, nq, L per column)
        self.select_rounds = []           # (rnd, R per column, whether a live run crosses a multiple of 256 ranks)

    def quantile_hist_chunk(self, x, state, nq, rnd, hist, first=False):
        from test_quantile_host import _state_views

        if rnd > 0 and first:
            head, _, _ = _state_views(state, int(x.shape[1]), nq)
            self.hist_rounds.append((rnd, nq, head["L"].copy()))
        super().quantile_hist_chunk(x, state, nq, rnd, hist, first)

    def quantile_select_step(self, hist, state, d, nq, rnd, dtype, qf):
        from test_quantile_host import _state_views

        super().quantile_select_step(hist, state, d, nq, rnd, dtype, qf)
        head, rec, _ = _state_views(state, d, nq)
        cross = []
        for j in range(d):
            slot = rec["slot"][j, : int(head["R"][j])]
            i = np.arange(256, len(slot), 256)
            cross.append(bool(head["L"][j] > 0 and (slot[i] == slot[i - 1]).any()))
        self.select_rounds.append((rnd, head["R"].copy(), np.array(cross)))


def device_data(be, case, rows=None):
    from dask_ml_b200.engine import DeviceData

    t = case.tensor()
    rows = rows or case.n
    return DeviceData([be.to_device(t[i:i + rows], t.dtype) for i in range(0, case.n, rows)], be)


def check_order_statistics(case, nq, missing, lo, hi, m):
    """lo / hi against np.sort of each column's valid values at the floor and floor + 1 ranks (as values: the sign of a
    zero may differ, numpy's own order of -0.0 and +0.0 being unspecified)."""
    v = case.values()
    qf = sc.references(nq)
    for j in range(case.d):
        col = v[:, j]
        ok = ~np.isnan(col) if missing is None else ~np.isnan(col) & (col != missing)
        s = np.sort(col[ok])
        assert m[j] == len(s), (case, j)
        if len(s) == 0:
            continue
        vi = (len(s) - 1.0) * qf
        top = vi >= len(s) - 1.0
        rlo = np.where(top, len(s) - 1, np.floor(vi)).astype(np.int64)
        rhi = np.where(top, len(s) - 1, np.floor(vi) + 1).astype(np.int64)
        np.testing.assert_array_equal(lo[j], s[rlo], err_msg="%r column %d lo" % (case, j))
        np.testing.assert_array_equal(hi[j], s[rhi], err_msg="%r column %d hi" % (case, j))


@pytest.fixture(scope="module")
def plan_runs():
    """order_statistics of every entry of the replay plan through the recording backend: (backend, failures)."""
    from dask_ml_b200.preprocessing.data import order_statistics

    be = RecordingBackend()
    fails = []
    for name, dt, d, nq, missing in sc.plan():
        case = sc.make(name, dt, d, nq)
        n_hist = len(be.hist_rounds)
        lo, hi, m = order_statistics(device_data(be, case), sc.references(nq), missing=missing)
        be.hist_rounds[n_hist:] = [(dt,) + r for r in be.hist_rounds[n_hist:]]
        try:
            check_order_statistics(case, nq, missing, lo, hi, m)
        except AssertionError as e:
            fails.append("%r nq=%d missing=%r: %s" % (case, nq, missing, str(e)[:400]))
    return be, fails


def test_plan_order_statistics(plan_runs):
    _, fails = plan_runs
    assert not fails, "\n".join(fails)


def test_plan_coverage(plan_runs):
    """The plan's cases reach the live-list regimes the GPU replay pins; a change to the cases that loses one fails
    here instead of leaving that regime unchecked."""
    be, _ = plan_runs
    rounds = be.hist_rounds
    for dt in sc.DTYPES:                                       # round 0 fills all 256 bins at the target ranks
        assert any(r[0] == dt and r[1] == 1 and (r[3] == 256).any() for r in rounds), dt
    assert any(staged(dt, rnd, nq) and (L > 256).any() for dt, rnd, nq, L in rounds)
    assert any(not staged(dt, rnd, nq) and (L >= 1000).any() for dt, rnd, nq, L in rounds if rnd > 0)
    for dt in ("f32", "f64"):                                  # n_q = 10000 drives rounds 2+ to global memory
        assert any(r[0] == dt and r[1] >= 2 and not staged(dt, r[1], r[2]) and (r[3] >= 1000).any() for r in rounds)
    assert any((R > 256).any() and cross.any() for _, R, cross in be.select_rounds)


def test_staging_rule_restated():
    """The restated rule at its edges: fp32 stages up to cap 3072, fp64 up to 3072, bf16 up to 1536."""
    assert staged("f32", 2, 1536) and not staged("f32", 2, 1537)
    assert staged("f64", 2, 1536) and not staged("f64", 2, 1537)
    assert staged("bf16", 1, 10000) and not staged("f32", 0, 1)
    assert not staged("f32", 2, 10000) and staged("f32", 1, 10000)


@pytest.fixture
def cpu_backend(monkeypatch):
    from dask_ml_b200.cluster import k_means as km

    monkeypatch.setattr(km, "_BACKEND_FACTORY", ImputeOracleBackend)
    return ImputeOracleBackend()


@pytest.mark.parametrize("dt", sc.DTYPES)
@pytest.mark.parametrize("name", ["full_range", "one_prefix", "carry", "zero_carry", "boundary", "specials"])
def test_quantiles_match_numpy(cpu_backend, name, dt):
    from dask_ml_b200.preprocessing import QuantileTransformer

    for nq in (57, 1000):
        case = sc.make(name, dt, sc.sector(dt) + 1, nq)
        qt = QuantileTransformer(n_quantiles=nq, subsample=10 ** 6).fit(device_data(cpu_backend, case, 1777))
        with np.errstate(all="ignore"):
            want = np.percentile(case.values(), qt.references_ * 100, axis=0)
        np.testing.assert_array_equal(qt.quantiles_, want, err_msg="%r nq=%d" % (case, nq))


QSETS = [(25, 75), (0, 100), (50, 50), (0.1, 99.9)]


def robust_cases():
    return [(name, dt) for dt in sc.DTYPES for name in ("full_range", "one_prefix", "carry", "zero_carry", "boundary",
                                                         "specials")]


@pytest.mark.parametrize("name,dt", robust_cases())
def test_percentiles_and_robust_scaler(cpu_backend, name, dt):
    """percentiles (the bkm_radix_* selection) equal np.nanpercentile of every NaN-free column and are NaN for a column
    with a NaN (numpy's percentile, as the reference's da.percentile); RobustScaler's scale_ equals scikit-learn's and
    its center_ numpy's 50th percentile of the list [25, 50, 75] wherever scikit-learn accepts the data (no inf).
    scikit-learn's center_ is np.nanmedian, the mean of the two middle values, which can round differently from the
    percentile's interpolation that the reference defines."""
    from dask_ml_b200.preprocessing import RobustScaler
    from dask_ml_b200.preprocessing.data import percentiles

    case = sc.make(name, dt, 3 * sc.sector(dt) + 1, 57)
    X = device_data(cpu_backend, case, 2500)
    v = case.values()
    nan = np.isnan(v).any(0)
    for q in QSETS:
        got = percentiles(X, list(q))
        with np.errstate(all="ignore"), warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            want = np.stack([np.nanpercentile(v[:, j], q) for j in range(case.d)])
        want[nan] = np.nan
        np.testing.assert_array_equal(got, want, err_msg="%r q=%s" % (case, q))
    fin = np.isfinite(v).all(0)
    if not fin.any():
        return
    rs = RobustScaler().fit(X)
    sk = sklearn.preprocessing.RobustScaler().fit(v[:, fin])
    np.testing.assert_array_equal(rs.scale_[fin], sk.scale_, err_msg=repr(case))
    with np.errstate(all="ignore"):
        want = np.percentile(v[:, fin], [25.0, 50.0, 75.0], axis=0)       # a list: numpy's percentile in float64
    np.testing.assert_array_equal(rs.center_[fin], want[1], err_msg=repr(case))


def sk_imputer(v, strategy, missing):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return sklearn.impute.SimpleImputer(strategy=strategy, missing_values=missing).fit(v)


def imputer_cases():
    out = []
    for dt in sc.DTYPES:
        for name in ("boundary", "zero_carry", "masked", "masked_zero", "specials", "carry"):
            out.append((name, dt, "median"))
        for name in ("mode_ties", "mode_many", "masked", "masked_zero", "specials", "zero_carry"):
            out.append((name, dt, "most_frequent"))
    return out


@pytest.mark.parametrize("name,dt,strategy", imputer_cases())
def test_imputer_statistics_match_scikit_learn(cpu_backend, name, dt, strategy):
    """median and most_frequent statistics_ equal scikit-learn's on the same values (a zero compares equal to either
    sign: the mode's zero is +0.0 here, scikit-learn's the first zero it meets)."""
    from dask_ml_b200.impute import SimpleImputer

    case = sc.make(name, dt, sc.sector(dt) + 1)
    v = case.values()
    missing = np.nan if case.missing is None else case.missing
    if not np.isnan(missing) and np.isnan(v).any():
        return
    fin = ~np.isinf(v).any(0)                                 # scikit-learn refuses inf
    v, case.bits = v[:, fin], case.bits[:, fin]
    got = SimpleImputer(strategy=strategy, missing_values=missing).fit(device_data(cpu_backend, case, 1500))
    want = sk_imputer(v, strategy, missing)
    np.testing.assert_array_equal(got.statistics_.astype(np.float64), want.statistics_.astype(np.float64),
                                  err_msg=repr(case))


def test_column_groups_split_the_selection(cpu_backend, monkeypatch):
    """A lowered HIST_BUDGET runs the selection in column groups of two with the same order statistics."""
    from dask_ml_b200.preprocessing import data as pp

    case = sc.make("full_range", "f32", 3 * sc.sector("f32") + 1, 1000)
    want = pp.order_statistics(device_data(cpu_backend, case, 4000), sc.references(1000))
    n0 = cpu_backend.launch_count()
    monkeypatch.setattr(pp, "HIST_BUDGET", 2 * 2000 * 256 * 8)
    got = pp.order_statistics(device_data(cpu_backend, case, 4000), sc.references(1000))
    assert cpu_backend.launch_count() - n0 == 13 * 4 * (5 + 1)          # 13 groups, 4 rounds, 5 chunks + a select
    for a, b in zip(got, want):
        np.testing.assert_array_equal(a, b)
    check_order_statistics(case, 1000, None, *got)
