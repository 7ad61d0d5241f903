"""The linear models on sparse X without a GPU: the estimators' sparse intake, the sparse passes' host plumbing, the
solver selection above the Newton bound and 2 ranks over gloo, on a CPU backend whose four sparse passes are float64
scipy restatements.  Sparse fits are checked against the dense fit of ``X.toarray()`` and against scikit-learn."""
import os
import socket
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_glm_host import CASES, GLMOracleBackend, _est, _np, _rel, glm_terms, sk_ref  # noqa: E402


def _csr(blk, d, dtype=np.float64):
    crow, col, val, n = blk
    v = val.numpy().astype(dtype)
    return sp.csr_matrix((v, col.numpy(), crow.numpy()), shape=(n, d))


def _canonical(blk, d):
    crow, col = blk[0].numpy(), blk[1].numpy()
    if ((col < 0) | (col >= d)).any():
        return False
    inner = np.ones(len(col), dtype=bool)
    inner[crow[1:-1]] = False                      # the first entry of each row after the first
    if len(col) == 0:
        return True
    return bool((np.diff(col)[inner[1:]] > 0).all())


class SparseOracleBackend(GLMOracleBackend):
    """The CPU checker backend plus float64 scipy restatements of the four sparse passes."""

    def glm_csr_pass_chunk(self, blk, d, y, beta, family, mode, r=None, w=None, grad=None, hrow=None, out=None,
                           first=False):
        self.launches += 1
        X = _csr(blk, d)
        b = beta.numpy()
        eta = X @ b[:-1] + b[-1]
        mu, loss, rr, ww = glm_terms(family, eta, y.numpy() if y is not None else np.zeros_like(eta))
        if mode >= 2:
            out.copy_(torch.from_numpy(mu if mode == 2 else (mu > 0.5).astype(np.uint8)))
            return
        r.copy_(torch.from_numpy(rr))
        tail = torch.tensor([rr.sum(), loss.sum()], dtype=torch.float64)
        grad[d:d + 2].copy_(tail) if first else grad[d:d + 2].add_(tail)
        if mode == 1:
            w.copy_(torch.from_numpy(ww))
            hrow[d] = ww.sum() if first else hrow[d] + ww.sum()

    def csr_transpose_chunk(self, blk, d):
        self.launches += 1
        ok = _canonical(blk, d)
        C = _csr(blk, d, blk[2].numpy().dtype).tocsc() if ok else sp.csc_matrix((blk[3], d))
        C.sort_indices()
        plan = torch.tensor([0 if ok else 1, 0, 0, 0], dtype=torch.int64)
        return (torch.from_numpy(C.indptr.astype(np.int64)), torch.from_numpy(C.indices.astype(np.int32)),
                torch.from_numpy(C.data.astype(blk[2].numpy().dtype)), plan)

    def csc_matvec_chunk(self, csc, d, v1, out1, v2=None, out2=None, first=False):
        self.launches += 1
        colptr, rows, vals, _plan = csc
        n = max(int(v1.numel()), int(rows.max()) + 1 if rows.numel() else 0)
        C = sp.csc_matrix((vals.numpy().astype(np.float64), rows.numpy(), colptr.numpy()), shape=(n, d))
        for v, o in ((v1, out1), (v2, out2)):
            if v is not None:
                g = torch.from_numpy(C.T @ v.numpy())
                o[:d].copy_(g) if first else o[:d].add_(g)

    def gram_weighted_csr_chunk(self, blk, csc, d, w, gram, n_slots, first=False):
        self.launches += 1
        X = _csr(blk, d)
        G = torch.from_numpy((X.T @ sp.diags(w.numpy()) @ X).toarray())
        gram.copy_(G) if first else gram.add_(G)


@pytest.fixture
def cpu_backend(monkeypatch):
    from dask_ml_b200.cluster import k_means as km

    monkeypatch.setattr(km, "_BACKEND_FACTORY", SparseOracleBackend)


def make_sparse(family, n=600, d=8, density=0.35, seed=0):
    """Canonical CSR X (float64, some rows empty) and y of the family."""
    rng = np.random.RandomState(seed)
    X = sp.random(n, d, density=density, format="csr", random_state=rng, data_rvs=rng.standard_normal)
    X[5] = 0
    X.eliminate_zeros()
    X.sort_indices()
    beta = rng.uniform(-0.6, 0.6, d)
    eta = X @ beta + 0.3
    if family == "logistic":
        y = (rng.uniform(size=n) < 1 / (1 + np.exp(-eta))).astype(np.float64)
    elif family == "normal":
        y = eta + 0.5 * rng.standard_normal(n)
    else:
        y = rng.poisson(np.exp(eta)).astype(np.float64)
    return X, y


def torch_csr(m, index_dtype=torch.int64, values=None):
    v = torch.from_numpy(np.ascontiguousarray(m.data)) if values is None else values
    return torch.sparse_csr_tensor(torch.from_numpy(m.indptr).to(index_dtype), torch.from_numpy(m.indices).to(index_dtype),
                                   v, size=m.shape)


def chunked(m, rows):
    from dask_ml_b200 import ChunkedArray

    return ChunkedArray([torch_csr(m[i:i + rows]) for i in range(0, m.shape[0], rows)])


TIGHT = {"newton": 1e-12, "admm": 1e-12, "lbfgs": 1e-12, "proximal_grad": 1e-13, "gradient_descent": 1e-15}


def fit(family, penalty, solver, X, y, fit_intercept=True, C=0.7):
    kw = {"factr": 10.0} if solver == "lbfgs" else None
    return _est(family, penalty=penalty or "l2", solver=solver, C=C, tol=TIGHT[solver], max_iter=20000,
                fit_intercept=fit_intercept, solver_kwargs=kw).fit(X, y)


def _beta(est):
    return np.append(est.coef_, est.intercept_) if hasattr(est, "intercept_") else est.coef_


@pytest.mark.parametrize("fit_intercept", [True, False])
@pytest.mark.parametrize("family,penalty,solver", CASES)
def test_sparse_fit_matches_dense_and_sklearn(cpu_backend, family, penalty, solver, fit_intercept):
    X, y = make_sparse(family)
    s = fit(family, penalty, solver, chunked(X, 250), y, fit_intercept)
    dn = fit(family, penalty, solver, X.toarray(), y, fit_intercept)
    # Newton-type solvers take the same iterates up to summation order; first-order line searches may branch on
    # last-bit differences, so those fits agree to their tolerance
    assert _rel(_beta(s), _beta(dn)) < (1e-8 if solver in ("newton", "admm") else 1e-6)
    if fit_intercept:
        assert _rel(_beta(s), sk_ref(family, penalty, 0.7, X.toarray(), y)) < 1e-6
    Xd = X.toarray()
    eta = Xd @ s.coef_ + (s.intercept_ if fit_intercept else 0.0)
    if family == "logistic":
        np.testing.assert_allclose(_np(s.predict_proba(X)), 1 / (1 + np.exp(-eta)), rtol=1e-12)
        np.testing.assert_array_equal(_np(s.predict(X)), 1 / (1 + np.exp(-eta)) > 0.5)
        assert s.score(X, y) == pytest.approx(np.mean(y == (1 / (1 + np.exp(-eta)) > 0.5)), abs=0)
    elif family == "normal":
        np.testing.assert_allclose(_np(s.predict(X)), eta, rtol=1e-11, atol=1e-12)
        assert s.score(X, y) == pytest.approx(np.mean((y - eta) ** 2), rel=1e-12)
    else:
        mu = np.exp(eta)
        np.testing.assert_allclose(_np(s.predict(X)), mu, rtol=1e-11)
        assert s.get_deviance(X, y) == pytest.approx(dn.get_deviance(Xd, y), rel=1e-8)


def test_sparse_predictions_are_chunked_like_x(cpu_backend):
    X, y = make_sparse("logistic")
    est = _est("logistic").fit(chunked(X, 250), y)
    p = est.predict_proba(chunked(X, 250))
    assert [int(b.shape[0]) for b in p.blocks] == [250, 250, 100]
    with pytest.raises(ValueError, match="X has 7 features, but LogisticRegression is expecting 8"):
        est.predict(X[:, :7])


def test_intake_forms(cpu_backend):
    from dask_ml_b200 import ChunkedArray

    X, y = make_sparse("poisson", seed=3)
    want = _beta(_est("poisson", tol=1e-12).fit(X.toarray(), y))
    coo = X.tocoo()
    dup = sp.coo_matrix((np.concatenate([coo.data / 2, coo.data / 2]), (np.concatenate([coo.row, coo.row]),
                        np.concatenate([coo.col, coo.col]))), shape=X.shape)     # duplicates summed at intake
    forms = [X, X.tocsc(), coo, dup, torch_csr(X), torch_csr(X, torch.int32), chunked(X, 170),
             ChunkedArray([torch_csr(X[i:i + 200], torch.int32) for i in range(0, 600, 200)])]
    for Xin in forms:
        got = _beta(_est("poisson", tol=1e-12).fit(Xin, y))
        np.testing.assert_allclose(got, want, rtol=1e-9)
    unsorted = X.copy()
    unsorted.has_sorted_indices = False
    unsorted.indices[:2], unsorted.data[:2] = unsorted.indices[1::-1].copy(), unsorted.data[1::-1].copy()
    unsorted.has_sorted_indices = False
    np.testing.assert_allclose(_beta(_est("poisson", tol=1e-12).fit(unsorted, y)), want, rtol=1e-9)  # scipy: sorted


@pytest.mark.parametrize("vdtype", [torch.uint8, torch.bool, torch.int32, torch.float32])
def test_value_dtypes(cpu_backend, vdtype):
    rng = np.random.RandomState(1)
    X = sp.random(500, 6, density=0.4, format="csr", random_state=rng)
    X.data[:] = 1.0
    y = (rng.uniform(size=500) < 0.5).astype(np.float64)
    want = _beta(_est("logistic", tol=1e-12).fit(X.toarray(), y))
    Xt = torch_csr(X, values=torch.from_numpy(X.data).to(vdtype))
    est = _est("logistic", tol=1e-12).fit(Xt, y)
    np.testing.assert_allclose(_beta(est), want, rtol=1e-9)
    np.testing.assert_array_equal(_np(est.predict(Xt)), _np(est.predict(X.toarray())))


def test_intake_errors(cpu_backend):
    from dask_ml_b200 import ChunkedArray

    X, y = make_sparse("logistic")
    mixed = ChunkedArray([torch_csr(X[:300]), torch.as_tensor(X[300:].toarray())])
    with pytest.raises(TypeError, match="mixes dense and sparse"):
        _est("logistic").fit(mixed, y)
    with pytest.raises(TypeError, match="float16"):
        _est("logistic").fit(torch_csr(X, values=torch.from_numpy(X.data).to(torch.float16)), y)
    bad = X[300:].copy()
    r = int(np.nonzero(np.diff(bad.indptr) >= 2)[0][0])
    k = bad.indptr[r]
    bad.indices[k], bad.indices[k + 1] = bad.indices[k + 1], bad.indices[k]
    blocks = ChunkedArray([torch_csr(X[:300]), torch_csr(bad)])
    with pytest.raises(ValueError, match="canonical CSR: the column indices of block 1"):
        _est("logistic").fit(blocks, y)
    nan = X.copy()
    nan.data[17] = np.nan
    with pytest.raises(ValueError, match="NaN, infinity"):
        _est("logistic").fit(chunked(nan, 250), y)
    with pytest.raises(ValueError, match="NaN, infinity"):
        _est("logistic", solver="lbfgs").fit(X, np.where(np.arange(600) == 3, np.inf, y))
    with pytest.raises(ValueError, match="inconsistent numbers of samples"):
        _est("logistic").fit(X, y[:-1])


def test_y_chunked_differently(cpu_backend):
    from dask_ml_b200 import ChunkedArray

    X, y = make_sparse("normal")
    base = _est("normal", tol=1e-12).fit(chunked(X, 250), y)
    for yy in (ChunkedArray.from_array(y, 77), torch.as_tensor(y), ChunkedArray.from_array(torch.as_tensor(y), 333)):
        np.testing.assert_allclose(_beta(_est("normal", tol=1e-12).fit(chunked(X, 250), yy)), _beta(base), rtol=1e-12)


def test_newton_bound(cpu_backend, monkeypatch):
    from dask_ml_b200.linear_model import glm

    X, y = make_sparse("logistic")
    monkeypatch.setattr(glm, "SPARSE_NEWTON_MAX_P", 8)       # p = 9 with the intercept
    with pytest.raises(ValueError, match="too large for sparse input.*'lbfgs', 'gradient_descent' or 'proximal_grad'"):
        _est("logistic", solver="newton").fit(X, y)
    assert _est("logistic", solver="newton", fit_intercept=False).fit(X, y).coef_.shape == (8,)   # p = 8: Newton
    est = _est("logistic", C=0.7, tol=1e-10, solver_kwargs={"factr": 10.0}).fit(X, y)             # admm / l2 -> lbfgs
    assert _rel(_beta(est), sk_ref("logistic", "l2", 0.7, X.toarray(), y)) < 1e-6
    calls = []
    orig = glm.lbfgs
    monkeypatch.setattr(glm, "lbfgs", lambda P, **kw: calls.append(kw) or orig(P, **kw))
    _est("logistic", tol=1e-5).fit(X, y)
    assert calls and calls[0]["tol"] == 1e-5 and calls[0]["regularizer"] == "l2"
    l1 = _est("logistic", penalty="l1", C=0.05, tol=1e-12, max_iter=5000).fit(X, y)             # admm / l1: unchanged
    ref = _est("logistic", penalty="l1", C=0.05, tol=1e-12, max_iter=5000, solver="proximal_grad").fit(X.toarray(), y)
    assert _rel(_beta(l1), _beta(ref)) < 1e-6


def test_launches_per_evaluation(monkeypatch):
    from dask_ml_b200.cluster import k_means as km

    X, y = make_sparse("logistic")
    be = SparseOracleBackend()
    monkeypatch.setattr(km, "_BACKEND_FACTORY", lambda: be)
    _est("logistic", solver="newton", tol=0.0, max_iter=2).fit(chunked(X, 250), y)
    # three transposes, then three passes per block per Newton evaluation (row, column, Gram), three evaluations
    assert be.launch_count() == 3 + 3 * 3 * 3


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


SHARDS = [(0, 250), (250, 600)]


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist

    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dask_ml_b200.cluster import k_means as km
        from test_glm_sparse_host import SparseOracleBackend, _beta, chunked, make_sparse

        km._BACKEND_FACTORY = SparseOracleBackend
        lo, hi = SHARDS[rank]
        res = {}
        for family, solver in (("logistic", "admm"), ("poisson", "lbfgs"), ("normal", "proximal_grad")):
            X, y = make_sparse(family)
            est = _est(family, solver=solver, penalty="l1" if solver == "proximal_grad" else "l2", tol=1e-12,
                       max_iter=5000).fit(chunked(X[lo:hi], 100), y[lo:hi])
            res[family] = _beta(est)
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **res)
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_ranks_equal_one_rank(tmp_path, cpu_backend):
    mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r = [np.load(tmp_path / ("rank%d.npz" % k)) for k in range(2)]
    for family, solver in (("logistic", "admm"), ("poisson", "lbfgs"), ("normal", "proximal_grad")):
        np.testing.assert_array_equal(r[0][family], r[1][family])
        X, y = make_sparse(family)
        one = _est(family, solver=solver, penalty="l1" if solver == "proximal_grad" else "l2", tol=1e-12,
                   max_iter=5000).fit(X, y)
        np.testing.assert_allclose(r[0][family], _beta(one), rtol=1e-7)
