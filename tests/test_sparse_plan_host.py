"""The sparse cases and the numpy restatement of the transpose's plan and the label sums (tests/sparse_cases.py), without
a GPU: the plan against scipy and against its bounds, the limits each case reaches (so that an edit to the cases cannot
quietly lose one), the restated label sums against Xᵀ·onehot, and the intake bound of the label-sum pass."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sparse_cases as sc  # noqa: E402

COLUMN_CASES = sorted(sc.column_cases())
ROW_CASES = sorted(sc.row_cases())
_cache = {}


def _pair(kind, name, dtype=np.float64, values="int"):
    key = (kind, name, np.dtype(dtype).name, values)
    if key not in _cache:
        _cache[key] = (sc.column_cases if kind == "col" else sc.row_cases)(dtype, values)[name]()
    return _cache[key]


def _plans(kind, name):
    return [sc.plan(m, m.shape[1]) for m in _pair(kind, name)]


@pytest.mark.parametrize("name", COLUMN_CASES)
def test_plan_matches_scipy_and_its_bounds(name):
    for m in _pair("col", name):
        d = m.shape[1]
        P = sc.plan(m, d)
        C = m.tocsc()
        C.sort_indices()
        np.testing.assert_array_equal(P.colptr, C.indptr)
        np.testing.assert_array_equal(P.rows, C.indices)
        np.testing.assert_array_equal(P.vals, C.data)
        T = int(P.status[1])
        assert T == len(P.seg_col) <= sc.seg_cap(d, m.nnz)
        assert P.status[3] == P.lens.max()
        # the segments tile each column in order, at most SEG entries each
        assert (P.seg_e1 - P.seg_e0 <= sc.SEG).all() and (P.seg_e1 >= P.seg_e0).all()
        np.testing.assert_array_equal(P.seg_e0[1:][P.seg_col[1:] == P.seg_col[:-1]],
                                      P.seg_e1[:-1][P.seg_col[1:] == P.seg_col[:-1]])
        np.testing.assert_array_equal(np.bincount(P.seg_col, weights=P.seg_e1 - P.seg_e0, minlength=d), P.lens)
        # the slots of multi-segment columns are distinct and inside the slot area
        sl = P.seg_slot[P.seg_slot >= 0]
        assert len(np.unique(sl)) == len(sl)
        assert sl.max(initial=-1) < sc.slot_rows(P)
        # one Gram slot per run of a column of several runs, distinct, inside plan[2]
        rs = P.run_slot[P.run_slot >= 0]
        np.testing.assert_array_equal(np.sort(rs), np.arange(P.status[2]))


def test_packed_multiseg_fills_the_slot_formula():
    """Columns of SEG + 1 entries: column j's slots are 2 j and 2 j + 1, so the last slot is 2 d - 1, two rows below
    the slot area 2 (nnz / SEG + 1)."""
    m = sc.packed_multiseg(40)
    P = sc.plan(m, 40)
    assert (P.nseg == 2).all()
    np.testing.assert_array_equal(P.seg_slot, np.arange(80))
    assert P.seg_slot.max() == 2 * 40 - 1 and sc.slot_rows(P) == 2 * 40 + 2
    # halving the stride (s0 - j) + (t - s0) makes neighbouring columns share a slot
    j = P.seg_col.astype(np.int64)
    s0 = P.seg_off[j]
    bad = (s0 - j) + (np.arange(len(j)) - s0)
    assert len(np.unique(bad)) < len(bad)


def test_column_cases_reach_the_plan_limits():
    segs, runs = set(), set()
    for name in COLUMN_CASES:
        for P in _plans("col", name):
            segs |= set(P.nseg.tolist())
            runs |= set(((P.nseg + sc.GS - 1) // sc.GS).tolist())
    assert {1, 2, 3, 33, 97} <= segs
    assert {1, 2, 3, 4} <= runs
    m = _pair("col", "edges")[0]
    lens = np.diff(m.tocsc().indptr)
    for L in (0, 1, 2047, 2048, 2049, 4097, 65535, 65536, 65537, 131073, 3 * 65536 + 1):
        assert L in lens
    assert lens[0] == 3 * 65536 + 1 and lens[-1] == 131073                   # long columns at j = 0 and d - 1
    assert (lens[1:3] == 0).all()                                            # next to empty ones
    assert (np.diff(_pair("col", "edges")[1].tocsc().indptr)[-5:] == 0).all()   # trailing empty columns
    # the Gram widths: 8, 8, 7 and 3 warps, each case with columns of several runs
    assert [sc.gram_warps(d) for d in sc.GRAM_D] == [8, 8, 7, 3]
    for d in sc.GRAM_D:
        name = "edges" if d == 18 else "gram%d" % d
        for P in _plans("col", name):
            assert P.d == d and P.status[2] >= 9 and P.nseg.max() == 97


def test_row_cases_reach_the_row_limits():
    G = {}
    for name in ROW_CASES:
        m = _pair("row", name)[0]
        G[name] = sc.row_group(m.shape[0], m.nnz)
    assert set(G.values()) == {4, 8, 16, 32}
    # each threshold crossed: exactly at t, and one entry above it
    for t, lo, hi in ((6, 4, 8), (12, 8, 16), (24, 16, 32)):
        assert G["mean%d+0" % t] == lo and G["mean%d+1" % t] == hi
        assert _pair("row", "mean%d+0" % t)[0].nnz == 1000 * t
    m = _pair("row", "skewed")[0]
    assert G["skewed"] == 4 and np.diff(m.indptr).max() == 100000
    lens = set(np.diff(_pair("row", "rows")[0].indptr).tolist())
    assert set(range(66)) | {1024, 1025, 2048} <= lens
    # the column tiles of the row-gather passes
    assert {sc.col_tile(l) for l in sc.L_PANEL} == {1, 2, 4}
    assert {sc.col_tile(k) for k in sc.K_ASSIGN} == {1, 2, 4}
    assert {sc.col_tile(k) for k in sc.K_NB} == {1, 2, 4}
    assert max(sc.col_tiles(l) for l in sc.L_PANEL) == 3
    assert min(sc.L_EMBED) > 128
    assert [sc.colsum_windows(l) for l in sc.L_COLSUM] == [1, 2, 3]


def test_label_sum_widths():
    assert [sc.label_sums_warps(k) for k in sc.K_LABEL] == [8, 8, 8, 8, 7, 1]
    assert sc.label_sums_warps(sc.MAX_LABEL_SUM_K + 1) == 0                # the pass refuses it


@pytest.mark.parametrize("values", ["int", "rand"])
@pytest.mark.parametrize("name", COLUMN_CASES)
def test_restated_label_sums_match_the_product(name, values):
    m1, m2 = _pair("col", name, values=values)
    d = m1.shape[1]
    P1, P2 = sc.plan(m1, d), sc.plan(m2, d)
    rng = np.random.RandomState(3)
    k = 33
    l1, l2 = rng.randint(-1, k, m1.shape[0]), rng.randint(0, k, m2.shape[0])
    w1 = rng.randint(1, 8, m1.shape[0]) / 4.0
    got = sc.label_sums(P2, l2, k, prev=sc.label_sums(P1, l1, k))
    want = (m1.T @ sc.onehot(l1, k)).toarray() + (m2.T @ sc.onehot(l2, k)).toarray()
    gotw = sc.label_sums(P1, l1, k, w=w1, binarize=1.5)
    A = (m1 > 1.5).astype(np.float64)
    wantw = (A.T @ sc.onehot(l1, k, w1)).toarray()
    if values == "int":
        np.testing.assert_array_equal(got, want)
        np.testing.assert_array_equal(gotw, wantw)
    else:
        scale = (abs(m1).T @ sc.onehot(l1, k)).toarray() + (abs(m2).T @ sc.onehot(l2, k)).toarray()
        assert (np.abs(got - want) <= 1e-13 * scale).all()
        np.testing.assert_array_equal(gotw, wantw)          # binarised with dyadic weights: exact either way


def test_restated_label_sums_follow_row_order():
    """Within a segment the sums run in row order, and a column's segments are added in segment order: 1 + 2^53 - 2^53
    is 0 in that order and 1 in any pairwise one."""
    n = 2 * sc.SEG + 5
    vals = np.zeros(n)
    vals[:3] = [1.0, 2.0 ** 53, -(2.0 ** 53)]
    vals[sc.SEG + 1:sc.SEG + 4] = [1.0, 2.0 ** 53, -(2.0 ** 53)]
    vals[vals == 0] = 0.5 ** 60
    m = sp.csr_matrix(sp.coo_matrix((vals, (np.arange(n), np.zeros(n, np.int64))), shape=(n, 1)))
    P = sc.plan(m, 1)
    assert P.nseg[0] == 3
    lab = np.zeros(n, np.int64)
    want = 0.0
    for s in range(3):
        acc = 0.0
        for v in vals[s * sc.SEG:(s + 1) * sc.SEG]:
            acc += v
        want += acc
    assert sc.label_sums(P, lab, 1)[0, 0] == want
    assert want != np.sum(vals)


# ---------------------------------------------------------------------------------------------------------------------
# the intake bound of the label-sum pass
# ---------------------------------------------------------------------------------------------------------------------
def _small_csr():
    return sp.random(40, 6, density=0.5, format="csr", random_state=0) + sp.eye(40, 6, format="csr")


def test_sparse_kmeans_refuses_more_clusters_than_the_label_sums_take(monkeypatch):
    from dask_ml_b200._sparse import MAX_LABEL_SUM_CLASSES
    from dask_ml_b200.cluster import KMeans, k_means as km
    from dask_ml_b200.cluster.k_means import k_means
    from test_kmeans_sparse_host import KMeansSparseOracleBackend

    assert MAX_LABEL_SUM_CLASSES == sc.MAX_LABEL_SUM_K
    monkeypatch.setattr(km, "_BACKEND_FACTORY", KMeansSparseOracleBackend)
    X = _small_csr()
    with pytest.raises(ValueError, match="at most 25600 clusters, got 25601"):
        KMeans(n_clusters=25601, init="random", random_state=0).fit(X)
    with pytest.raises(ValueError, match="at most 25600 clusters"):
        k_means(X, 25601, init="random", random_state=0)
    KMeans(n_clusters=3, init="random", random_state=0, max_iter=2).fit(X)            # within the bound: runs


def test_sparse_minibatch_refuses_more_clusters_than_the_label_sums_take(monkeypatch):
    from dask_ml_b200.cluster import PartialMiniBatchKMeans, k_means as km
    from test_minibatch_host import MiniBatchChecker

    monkeypatch.setattr(km, "_BACKEND_FACTORY", MiniBatchChecker)
    with pytest.raises(ValueError, match="at most 25600 clusters, got 25601"):
        PartialMiniBatchKMeans(n_clusters=25601).partial_fit(_small_csr())
    assert not hasattr(PartialMiniBatchKMeans(n_clusters=25601), "cluster_centers_")
    # dense rows take the dense passes: the bound does not apply (this fails later, on the batch size)
    with pytest.raises(ValueError, match="should be >= n_clusters"):
        PartialMiniBatchKMeans(n_clusters=25601).partial_fit(_small_csr().toarray())


def test_sparse_naive_bayes_refuses_more_classes_than_the_label_sums_take(monkeypatch):
    from dask_ml_b200.cluster import k_means as km
    from dask_ml_b200.naive_bayes import PartialBernoulliNB, PartialMultinomialNB
    from test_partial_nb_host import NBChecker

    monkeypatch.setattr(km, "_BACKEND_FACTORY", NBChecker)
    X = _small_csr()
    y = np.arange(40) % 3
    many, few = np.arange(25601), np.arange(3)
    for cls in (PartialMultinomialNB, PartialBernoulliNB):
        est = cls(classes=many)
        with pytest.raises(ValueError, match="at most 25600 classes, got 25601"):
            est.partial_fit(X, y, classes=many)
        assert not hasattr(est, "classes_")                  # refused before any state was set
        with pytest.raises(ValueError, match="at most 25600 classes"):
            cls(classes=many).fit(X, y)
        est = cls(classes=few).partial_fit(X, y, classes=few)
        est.partial_fit(X, y)
        # dense rows take the dense count pass, which has no such bound
        cls(classes=many).partial_fit(X.toarray(), y, classes=many)
