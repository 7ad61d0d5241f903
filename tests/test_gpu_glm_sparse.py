"""The sparse passes of the linear models on the H100: the CSR row pass, the transpose, the column pass and the sparse
weighted Gram against float64 scipy for float32 and float64 values, bit-identical repeats, edge shapes (n = 1, d = 1,
d = 2^20, nnz = 0, empty rows, a column in every row, p at the Newton bound, ragged blocks), and the estimators fed by
OneHotEncoder and HashingVectorizer."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_glm_host import _est, _np, glm_terms  # noqa: E402
from test_glm_sparse_host import SparseOracleBackend, _beta, make_sparse, torch_csr  # noqa: E402

pytestmark = pytest.mark.gpu

DT = {"f32": (torch.float32, np.float32), "f64": (torch.float64, np.float64)}


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


def rand_csr(n, d, density, dt, seed, heavy=None):
    """Canonical CSR of n x d in the numpy dtype of ``dt`` (some rows empty); ``heavy`` columns present in every row."""
    rng = np.random.RandomState(seed)
    k = int(round(n * d * density))                # sampled coordinates: sp.random would permute all n d cells
    m = sp.csr_matrix((rng.standard_normal(k), (rng.randint(0, n, k), rng.randint(0, d, k))), shape=(n, d))
    if heavy is not None:
        cols = m.tocsc()
        cols = [sp.csc_matrix(rng.standard_normal((n, 1)) + 3.0) if j in heavy else cols[:, j] for j in range(d)]
        m = sp.hstack(cols, format="csr")
    m = m.astype(DT[dt][1])
    m.sum_duplicates()
    m.sort_indices()
    return m


def device_blk(be, m):
    return (torch.as_tensor(m.indptr.astype(np.int64)).to(be.device), torch.as_tensor(m.indices.astype(np.int64)).to(be.device),
            torch.as_tensor(m.data).to(be.device), m.shape[0])


def run_passes(be, blk, d, y, beta, family):
    n = blk[3]
    dev = be.device
    csc = be.csr_transpose_chunk(blk, d)
    st = csc[3][:4].cpu().numpy()
    grad = torch.full((d + 2,), 7.0, dtype=torch.float64, device=dev)
    hrow = torch.full((d + 1,), 7.0, dtype=torch.float64, device=dev)
    r = torch.empty(n, dtype=torch.float64, device=dev)
    w = torch.empty(n, dtype=torch.float64, device=dev)
    be.glm_csr_pass_chunk(blk, d, y, beta, family, 1, r=r, w=w, grad=grad, hrow=hrow, first=True)
    be.csc_matvec_chunk(csc, d, r, grad, v2=w, out2=hrow, first=True)
    g0 = torch.empty_like(grad)
    r0 = torch.empty_like(r)
    be.glm_csr_pass_chunk(blk, d, y, beta, family, 0, r=r0, grad=g0, first=True)
    be.csc_matvec_chunk(csc, d, r0, g0, first=True)
    G = None
    if d <= 4096:
        G = torch.full((d, d), 7.0, dtype=torch.float64, device=dev)
        be.gram_weighted_csr_chunk(blk, csc, d, w, G, int(st[2]), first=True)
    mu = torch.empty(n, dtype=torch.float64, device=dev)
    lab = torch.empty(n, dtype=torch.uint8, device=dev)
    be.glm_csr_pass_chunk(blk, d, None, beta, family, 2, out=mu)
    be.glm_csr_pass_chunk(blk, d, None, beta, family, 3, out=lab)
    torch.cuda.synchronize()
    out = [t.cpu().numpy() if t is not None else None for t in (grad, hrow, r, w, g0, mu, lab, G)]
    return out, [t.cpu().numpy() for t in csc[:3]], st


def check(be, m, family, seed=1, scale=1.0):
    n, d = m.shape
    rng = np.random.RandomState(seed)
    b = rng.standard_normal(d + 1) * scale / np.sqrt(max(1.0, m.getnnz() / max(n, 1)))
    y = {0: (rng.uniform(size=n) < 0.5) * 1.0, 1: rng.standard_normal(n), 2: rng.poisson(2.0, n) * 1.0}[family]
    blk = device_blk(be, m)
    yd, bd = torch.as_tensor(y).to(be.device), torch.as_tensor(b).to(be.device)
    got, csc, st = run_passes(be, blk, d, yd, bd, family)
    grad, hrow, r, w, g0, mu, lab, G = got
    X = m.astype(np.float64)
    eta = X @ b[:-1] + b[-1]
    mw, lw, rw, ww = glm_terms(family, eta, y)
    A = abs(X)
    tol = lambda s: 1e-13 * np.maximum(s, 1e-300)                      # noqa: E731
    assert st[0] == 0
    # the transpose, bit for bit
    C = m.tocsc()
    C.sort_indices()
    np.testing.assert_array_equal(csc[0], C.indptr)
    np.testing.assert_array_equal(csc[1], C.indices)
    np.testing.assert_array_equal(csc[2], C.data)
    # the row pass
    esc = A @ np.abs(b[:-1]) + abs(b[-1])
    np.testing.assert_allclose(mu, mw, rtol=1e-12, atol=1e-14 * (esc.max(initial=0) + 1))
    np.testing.assert_array_equal(lab.astype(bool), mu > 0.5)
    np.testing.assert_allclose(r, rw, rtol=1e-12, atol=1e-13 * (esc.max(initial=0) + 1) * max(1, abs(rw).max(initial=0)))
    np.testing.assert_allclose(w, ww, rtol=1e-12, atol=1e-300)
    for got_v, want_v in ((grad[d], rw.sum()), (grad[d + 1], lw.sum()), (hrow[d], ww.sum())):
        assert abs(got_v - want_v) <= 1e-12 * max(1.0, np.abs(rw).sum() + np.abs(lw).sum() + np.abs(ww).sum())
    # the column pass: within 1e-13 of X^T r at the scale of |X|^T |r|
    assert (np.abs(grad[:d] - X.T @ r) <= tol(A.T @ np.abs(r))).all()
    assert (np.abs(hrow[:d] - X.T @ w) <= tol(A.T @ np.abs(w))).all()
    np.testing.assert_array_equal(g0, grad)                          # the gradient half of the Newton pass
    if G is not None:
        want = (X.T @ sp.diags(w) @ X).toarray()
        assert (np.abs(G - want) <= tol((A.T @ sp.diags(np.abs(w)) @ A).toarray())).all()
    again, csc2, st2 = run_passes(be, blk, d, yd, bd, family)
    for a1, a2 in zip(got + csc, again + csc2):
        if a1 is not None:
            np.testing.assert_array_equal(a1, a2)                      # bit-identical repeat
    np.testing.assert_array_equal(st, st2)
    return st


@pytest.mark.parametrize("dt", ["f32", "f64"])
@pytest.mark.parametrize("family", [0, 1, 2])
@pytest.mark.parametrize("n,d,density", [(1, 5, 0.6), (300, 1, 0.5), (4099, 37, 0.1), (3000, 700, 0.05),
                                         (2000, 50, 0.6), (3000, 1024, 0.01)])
def test_passes_against_scipy(be, dt, family, n, d, density):
    check(be, rand_csr(n, d, density, dt, seed=n + d), family)


@pytest.mark.parametrize("dt", ["f32", "f64"])
def test_edge_shapes(be, dt):
    check(be, sp.csr_matrix((5, 9), dtype=DT[dt][1]), 0)                          # nnz = 0
    m = rand_csr(1000, 30, 0.2, dt, seed=2)
    m[100:400] = 0                                                                   # empty rows
    m.eliminate_zeros()
    check(be, m, 2)
    check(be, rand_csr(20000, 1 << 20, 3e-5, dt, seed=3), 0)                        # d = 2^20 (no Gram)


@pytest.mark.parametrize("dt", ["f32", "f64"])
def test_heavy_columns(be, dt):
    """Columns present in every row: the column pass and the Gram split them and fold the parts in order."""
    m = rand_csr(150000, 64, 0.02, dt, seed=4, heavy=[0, 17])
    st = check(be, m, 0, scale=0.3)
    assert st[3] == 150000 and st[2] > 0


def test_newton_bound_shape(be):
    check(be, rand_csr(3000, 4095, 0.002, "f32", seed=6), 1)                        # p = 4096 with the intercept


def test_noncanonical_flag(be):
    m = rand_csr(200, 10, 0.5, "f64", seed=7)
    k = int(m.indptr[np.nonzero(np.diff(m.indptr) >= 2)[0][0]])
    m.indices[k], m.indices[k + 1] = m.indices[k + 1], m.indices[k]
    csc = be.csr_transpose_chunk(device_blk(be, m), 10)
    assert int(csc[3][0].item()) != 0


def test_estimators_ragged_blocks_match_checker(monkeypatch):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import k_means as km

    X, y = make_sparse("poisson", n=5000, d=40)
    sizes = [0, 1, 1000, 37, 2962, 1000]
    off = np.cumsum([0] + sizes)
    blocks = ChunkedArray([torch_csr(X[off[i]:off[i + 1]].astype(np.float32)).cuda() for i in range(len(sizes))])
    got = {s: _beta(_est("poisson", solver=s, tol=1e-10).fit(blocks, y)) for s in ("admm", "lbfgs")}
    monkeypatch.setattr(km, "_BACKEND_FACTORY", SparseOracleBackend)
    Xf = X.astype(np.float32).astype(np.float64)
    for s, b in got.items():
        want = _beta(_est("poisson", solver=s, tol=1e-10).fit(Xf, y))
        np.testing.assert_allclose(b, want, rtol=1e-8)


def test_one_hot_to_logistic():
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.linear_model import LogisticRegression
    from dask_ml_b200.preprocessing import OneHotEncoder

    rng = np.random.RandomState(8)
    n = 200000
    Xc = torch.as_tensor(rng.randint(0, 12, (n, 4))).cuda()
    logit = (Xc[:, 0].double() - 5.5) / 3 + torch.where(Xc[:, 1] % 3 == 0, 1.0, -0.5).double()
    y = (torch.rand(n, generator=torch.Generator().manual_seed(0), dtype=torch.float64).cuda() < torch.sigmoid(logit))
    Xcc = ChunkedArray([Xc[i:i + 60000] for i in range(0, n, 60000)])
    yc = ChunkedArray([y[i:i + 60000].double() for i in range(0, n, 60000)])
    Xs = OneHotEncoder(sparse=True).fit_transform(Xcc)
    assert all(b.layout == torch.sparse_csr and b.is_cuda for b in Xs.blocks)
    Xd = OneHotEncoder(sparse=False).fit_transform(Xcc)
    a = LogisticRegression().fit(Xs, yc)
    b = LogisticRegression().fit(Xd, yc)
    np.testing.assert_allclose(a.coef_, b.coef_, rtol=1e-8, atol=1e-8 * np.abs(b.coef_).max())
    assert a.intercept_ == pytest.approx(b.intercept_, rel=1e-8)
    np.testing.assert_array_equal(_np(a.predict(Xs)), _np(b.predict(Xd)))


@pytest.mark.parametrize("family", ["logistic", "poisson"])
def test_hashed_text_matches_checker(monkeypatch, family):
    from dask_ml_b200.cluster import k_means as km
    from dask_ml_b200.feature_extraction import HashingVectorizer
    from test_text_host import chunked, word_docs

    docs = word_docs(3000, seed=9, vocab=400)
    X = HashingVectorizer(n_features=2 ** 18).transform(chunked(docs, 700))
    rng = np.random.RandomState(10)
    Xh = X.compute()
    eta = Xh @ rng.uniform(-1, 1, 2 ** 18) * 0.5
    y = (rng.uniform(size=len(docs)) < 1 / (1 + np.exp(-eta))) * 1.0 if family == "logistic" \
        else rng.poisson(np.exp(eta)) * 1.0
    kw = dict(solver="lbfgs", tol=1e-8, solver_kwargs={"factr": 10.0})
    got = _est(family, **kw).fit(X, y)
    monkeypatch.setattr(km, "_BACKEND_FACTORY", SparseOracleBackend)
    want = _est(family, **kw).fit(Xh, y)
    assert np.abs(_beta(got) - _beta(want)).max() <= 1e-6 * max(1.0, np.abs(_beta(want)).max())
