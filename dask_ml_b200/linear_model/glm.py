"""LogisticRegression, LinearRegression and PoissonRegression with the dask_ml.linear_model API, executed by the H100
engine.

Mirrors dask_ml/linear_model/glm.py (reference @ 0310a90), whose solvers live in dask-glm.  With beta = [coef,
intercept] and the ones column last, every solver minimises f(beta) = L(beta) + lambda R(beta), lambda = 1 / C (or
``solver_kwargs['lamduh']``), the intercept penalised as in the reference, R = 1/2 ||beta||^2 (l2) or ||beta||_1 (l1):

    family    L(beta)                     mu            gradient r_i = c (mu - y)    Newton weight w_i
    logistic  sum softplus(eta) - y eta   sigmoid(eta)  mu - y                       mu (1 - mu)
    normal    sum (y - eta)^2             eta           2 (mu - y)                   2
    poisson   sum exp(eta) - y eta        exp(eta)      mu - y                       mu

Each evaluation is one device pass per chunk and one all-reduce:

    gradient pass (bkm_glm_pass_chunk mode 0):          [sum r x | sum r | loss]            all-reduce of [g | loss]
    Newton pass   (bkm_glm_pass_chunk mode 1, then      [sum r x | sum r | loss], w_i,
                   bkm_gram_weighted_chunk with w_i):   [sum w x | sum w], sum w x x^T      all-reduce of [H | g | loss]

Sparse X (a ChunkedArray of torch sparse CSR blocks, one torch CSR tensor, or any scipy.sparse matrix) runs the same
solvers on the same objective; only the per-block calls change (``_SparsePasses``):

    gradient pass (bkm_glm_csr_pass_chunk mode 0, then bkm_csc_matvec_chunk with r_i over the block's transpose)
    Newton pass   (mode 1, the column pass with r_i and w_i, then bkm_gram_weighted_csr_chunk with w_i)

The transpose of each block is built on the first evaluation of a fit and kept for it.

The solvers run on the host in float64 (DESIGN.md A22): 'newton' (unregularised, Cholesky, least squares when it
fails, the step halved until the loss passes an Armijo test, stop at max |delta| < tol), 'lbfgs' (scipy's fmin_l_bfgs_b, pgtol = tol), 'gradient_descent' (unregularised,
Armijo backtracking, stop when the relative decrease of the loss is below tol), 'proximal_grad' (backtracking on the
quadratic bound, stop at max |delta beta| < tol (1 + max |beta|)).  'admm' is a documented deviation: penalised Newton
for l2, 'proximal_grad' for l1 -- the exact optimum that the reference's consensus ADMM approximates.  On sparse X with
more than ``SPARSE_NEWTON_MAX_P`` coefficients the (p, p) Hessian is not formed: 'newton' raises, and l2 'admm' runs
'lbfgs' on the same objective (pgtol = tol).

Unregularised logistic regression on separable data has no finite optimum: the coefficients grow until max_iter, as in
the reference.
"""
import numpy as np
import scipy.linalg
import torch
from scipy.optimize import fmin_l_bfgs_b
from sklearn.base import BaseEstimator
from sklearn.exceptions import NotFittedError

from .._sparse import _SparseData, _sparse_data, _sparse_values  # noqa: F401  (the sparse intake, shared)
from ..chunked import ChunkedArray, _is_torch
from ..cluster.k_means import _NONFINITE_MSG
from ..decomposition.pca import _device_data
from ..naive_bayes import _y_flat

LOGISTIC, NORMAL, POISSON = 0, 1, 2                # the kernel's family codes
_GRAD, _NEWTON, _PREDICT, _LABEL = 0, 1, 2, 3      # and its modes
_SOLVERS = {"admm", "proximal_grad", "lbfgs", "newton", "gradient_descent"}
SPARSE_NEWTON_MAX_P = 4096                         # the largest p = d (+ 1) whose Hessian sparse input forms


def _y_chunks(y, X, who):
    """y in any form GaussianNB takes -> float64 device chunks split to X's chunk rows (``DeviceData.chunk_offsets``)."""
    yf = _y_flat(y, who)
    if int(yf.shape[0]) != X.n_local:
        raise ValueError("Found input variables with inconsistent numbers of samples: [%d, %d]"
                         % (X.n_local, int(yf.shape[0])))
    t = yf if _is_torch(yf) else torch.as_tensor(np.ascontiguousarray(yf, dtype=np.float64))
    t = t.to(device=X.backend.device, dtype=torch.float64)
    off = X.chunk_offsets
    return [t[int(off[i]):int(off[i + 1])].contiguous() for i in range(len(off) - 1)]


class _Passes(object):
    """The device passes of one fit: gradient and Newton evaluations at beta (length d + 1 with an intercept, else
    d), each summed over every chunk and rank."""

    def __init__(self, X, ys, family, fit_intercept):
        self.X, self.ys, self.family = X, ys, family
        self.be, self.comm, self.d = X.backend, X.comm, X.d
        self.p = self.d + 1 if fit_intercept else self.d
        self.checked = False
        self.wbuf = None

    def _beta(self, b):
        full = np.zeros(self.d + 1)
        full[: self.p] = b
        return torch.as_tensor(full).to(self.be.device)

    def _scanned(self):
        """The 2-D parts of X that the non-finite scan reads, one per y chunk."""
        return self.X.chunks

    def _check(self, vals):
        """The first evaluation is at beta = 0, where every term is finite for finite X and y: a non-finite result
        there is a NaN or inf in X or y.  X is scanned only then, as PCA does."""
        if self.checked:
            return
        self.checked = True
        if np.isfinite(vals).all():
            return
        be = self.be
        flag = torch.zeros(1, dtype=torch.float64, device=be.device)
        for x, y in zip(self._scanned(), self.ys):
            flag += be.check_finite([x]).to(torch.float64)
            flag += (~torch.isfinite(y)).any().to(torch.float64)
        self.comm.allreduce_sum_(flag)
        if float(flag.item()) != 0.0:
            raise ValueError(_NONFINITE_MSG)
        raise ValueError("Input contains values too large for the float64 loss or gradient")

    def grad(self, b):
        """(loss, gradient of the loss) at b: one gradient pass per chunk, one all-reduce of [g | loss]."""
        d, be = self.d, self.be
        bd = self._beta(b)
        red = be.zeros((d + 2,), torch.float64)
        for i, x in enumerate(self.X.chunks):
            be.glm_pass_chunk(x, self.ys[i], bd, self.family, _GRAD, grad=red, first=i == 0)
        self.comm.allreduce_sum_(red)
        h = red.cpu().numpy()
        self._check(h)
        return float(h[d + 1]), h[: self.p].copy()

    def newton(self, b):
        """(loss, gradient, Hessian) at b: a Newton pass and a weighted Gram pass per chunk, one all-reduce of
        [H | g | loss]."""
        d, be = self.d, self.be
        bd = self._beta(b)
        red = be.zeros((d * d + 2 * d + 3,), torch.float64)
        G, hrow, grad = red[: d * d].view(d, d), red[d * d: d * d + d + 1], red[d * d + d + 1:]
        if self.wbuf is None:
            self.wbuf = be.empty((max([1] + list(self.X.chunk_rows)),), torch.float64)
        for i, x in enumerate(self.X.chunks):
            w = self.wbuf[: int(x.shape[0])]
            be.glm_pass_chunk(x, self.ys[i], bd, self.family, _NEWTON, grad=grad, hrow=hrow, w=w, first=i == 0)
            be.gram_weighted_chunk(x, w, G, first=i == 0)
        self.comm.allreduce_sum_(red)
        h = red.cpu().numpy()
        self._check(h)
        H = np.empty((d + 1, d + 1))
        H[:d, :d] = h[: d * d].reshape(d, d)
        H[d, :d] = H[:d, d] = h[d * d: d * d + d]
        H[d, d] = h[d * d + d]
        g = h[d * d + d + 1:]
        return float(g[d + 1]), g[: self.p].copy(), H[: self.p, : self.p].copy()


class _SparsePasses(_Passes):
    """``_Passes`` on sparse CSR blocks: the same evaluations, reduction buffers and all-reduces, each block's terms
    from the CSR row pass, the column pass over its transpose and (Newton) the sparse weighted Gram."""

    def __init__(self, X, ys, family, fit_intercept):
        super(_SparsePasses, self).__init__(X, ys, family, fit_intercept)
        self.rbuf = None

    def _scanned(self):
        return [b[2].view(-1, 1) for b in self.X.blocks]

    def _bufs(self, newton):
        rows = max([1] + self.X.chunk_rows)
        if self.rbuf is None:
            self.rbuf = self.be.empty((rows,), torch.float64)
        if newton and self.wbuf is None:
            self.wbuf = self.be.empty((rows,), torch.float64)

    def grad(self, b):
        d, be = self.d, self.be
        bd = self._beta(b)
        csc = self.X.transposes()
        self._bufs(False)
        red = be.zeros((d + 2,), torch.float64)
        for i, blk in enumerate(self.X.blocks):
            r = self.rbuf[: blk[3]]
            be.glm_csr_pass_chunk(blk, d, self.ys[i], bd, self.family, _GRAD, r=r, grad=red, first=i == 0)
            be.csc_matvec_chunk(csc[i], d, r, red, first=i == 0)
        self.comm.allreduce_sum_(red)
        h = red.cpu().numpy()
        self._check(h)
        return float(h[d + 1]), h[: self.p].copy()

    def newton(self, b):
        d, be = self.d, self.be
        bd = self._beta(b)
        csc = self.X.transposes()
        self._bufs(True)
        red = be.zeros((d * d + 2 * d + 3,), torch.float64)
        G, hrow, grad = red[: d * d].view(d, d), red[d * d: d * d + d + 1], red[d * d + d + 1:]
        for i, blk in enumerate(self.X.blocks):
            r, w = self.rbuf[: blk[3]], self.wbuf[: blk[3]]
            be.glm_csr_pass_chunk(blk, d, self.ys[i], bd, self.family, _NEWTON, r=r, w=w, grad=grad, hrow=hrow,
                                  first=i == 0)
            be.csc_matvec_chunk(csc[i], d, r, grad, v2=w, out2=hrow, first=i == 0)
            be.gram_weighted_csr_chunk(blk, csc[i], d, w, G, self.X.n_slots[i], first=i == 0)
        self.comm.allreduce_sum_(red)
        h = red.cpu().numpy()
        self._check(h)
        H = np.empty((d + 1, d + 1))
        H[:d, :d] = h[: d * d].reshape(d, d)
        H[d, :d] = H[:d, d] = h[d * d: d * d + d]
        H[d, d] = h[d * d + d]
        g = h[d * d + d + 1:]
        return float(g[d + 1]), g[: self.p].copy(), H[: self.p, : self.p].copy()


# -- regularisers: (value, gradient or subgradient, proximal operator of t R) ------------------------------------------
def _regularizer(name):
    if name == "l2":
        return (lambda b: 0.5 * float(b @ b)), (lambda b: b), (lambda v, t: v / (1.0 + t))
    if name == "l1":
        return ((lambda b: float(np.abs(b).sum())), np.sign,
                (lambda v, t: np.sign(v) * np.maximum(np.abs(v) - t, 0.0)))
    raise ValueError("'penalty' must be 'l1' or 'l2'. Got %r instead" % (name,))


# -- solvers (host, float64); every one starts at beta = 0 -------------------------------------------------------------
_MAX_HALVINGS = 40
def newton(P, max_iter=50, tol=1e-8, ridge=0.0, **_):
    """Damped Newton's method on f = L + ridge/2 ||beta||^2.  ``ridge`` > 0 is the l2 'admm' path; the 'newton' solver
    is unregularised (a ``lamduh`` in ``solver_kwargs`` lands in ``**_``, as dask-glm's newton ignores it).

    A full Newton step can overshoot badly: from beta = 0 on counts of mean m, the Poisson intercept jumps to about
    m - 1, where exp(eta) is astronomically large or +inf.  So the step is halved until f passes the Armijo test (a
    non-finite f never does).  The candidate is evaluated with a Newton pass, whose Hessian serves the next iteration
    when the full step is taken; each halving costs one gradient pass.  Stops when the full step has max |delta| < tol
    (taken without another pass) or after max_iter iterations."""
    b = np.zeros(P.p)
    loss, g, H = P.newton(b)
    for _k in range(int(max_iter)):
        f = loss + 0.5 * ridge * float(b @ b)
        g = g + ridge * b
        H = H + ridge * np.eye(P.p)
        try:
            delta = scipy.linalg.cho_solve(scipy.linalg.cho_factor(H), g)
        except (np.linalg.LinAlgError, ValueError):
            delta = np.linalg.lstsq(H, g, rcond=None)[0]
        if np.max(np.abs(delta), initial=0.0) < tol:
            return b - delta
        dec = max(float(g @ delta), 0.0)                 # the squared Newton decrement, g^T H^-1 g
        t, nb = 1.0, b - delta
        nl, ng, nH = P.newton(nb)
        for _j in range(_MAX_HALVINGS + 1):
            fn = nl + 0.5 * ridge * float(nb @ nb)
            # False for NaN / inf; the slack admits the rounding of f at the optimum
            if fn <= f - 1e-4 * t * dec + 1e-12 * abs(f):
                break
            if _j == _MAX_HALVINGS:
                return b                                 # no decrease along the Newton direction: stationary
            t *= 0.5
            nb = b - t * delta
            nl, ng = P.grad(nb)
            nH = None
        if nH is None:
            nl, ng, nH = P.newton(nb)
        b, loss, g, H = nb, nl, ng, nH
    return b


def lbfgs(P, max_iter=100, tol=1e-4, regularizer="l2", lamduh=1.0, factr=1e7, **_):
    """scipy's L-BFGS-B on L + lamduh R (the subgradient lamduh sign(beta) for l1); ``factr`` (scipy's relative
    decrease test, default as scipy's) may come from ``solver_kwargs``."""
    Rv, Rg, _prox = _regularizer(regularizer)

    def f(b):
        loss, g = P.grad(b)
        return loss + lamduh * Rv(b), g + lamduh * Rg(b)

    b, _f, _info = fmin_l_bfgs_b(f, np.zeros(P.p), pgtol=tol, maxiter=int(max_iter), factr=factr)
    return b


def gradient_descent(P, max_iter=100, tol=1e-8, **_):
    """Steepest descent on the unregularised loss with Armijo backtracking (step x 0.1 on the first iteration, x 0.5
    after, x 1.25 growth per accepted step); stops when the relative decrease of the loss is below tol."""
    b = np.zeros(P.p)
    loss, g = P.grad(b)
    t, mult = 1.0, 0.1
    for _k in range(int(max_iter)):
        gg = float(g @ g)
        if gg == 0.0:
            break
        for _j in range(100):
            nb = b - t * g
            nl, ng = P.grad(nb)
            if nl <= loss - 0.1 * t * gg:          # False for NaN / inf: back off
                break
            t *= mult
        else:
            break
        rel = (loss - nl) / max(abs(loss), abs(nl), 1e-300)
        b, loss, g = nb, nl, ng
        if rel < tol:
            break
        t *= 1.25
        mult = 0.5
    return b


def proximal_grad(P, max_iter=100, tol=1e-8, regularizer="l1", lamduh=1.0, **_):
    """Proximal gradient with backtracking on the quadratic upper bound of the loss; stops when
    max |delta beta| < tol (1 + max |beta|)."""
    _Rv, _Rg, prox = _regularizer(regularizer)
    b = np.zeros(P.p)
    loss, g = P.grad(b)
    t, mult = 1.0, 0.1
    for _k in range(int(max_iter)):
        for _j in range(100):
            nb = prox(b - t * g, t * lamduh)
            s = nb - b
            nl, ng = P.grad(nb)
            if nl <= loss + float(g @ s) + float(s @ s) / (2.0 * t):
                break
            t *= mult
        else:
            break
        step = np.max(np.abs(s), initial=0.0)
        b, loss, g = nb, nl, ng
        if step < tol * (1.0 + np.max(np.abs(b), initial=0.0)):
            break
        t *= 1.25
        mult = 0.5
    return b


def admm(P, max_iter=100, tol=1e-4, regularizer="l2", lamduh=1.0, **_):
    """The exact optimum the reference's consensus ADMM approximates: penalised Newton for l2, proximal_grad for l1."""
    _regularizer(regularizer)
    if regularizer == "l2":
        return newton(P, max_iter=max_iter, tol=tol, ridge=lamduh)
    return proximal_grad(P, max_iter=max_iter, tol=tol, regularizer=regularizer, lamduh=lamduh)


_SOLVER_FNS = {"admm": admm, "proximal_grad": proximal_grad, "lbfgs": lbfgs, "newton": newton,
               "gradient_descent": gradient_descent}


class _GLM(BaseEstimator):
    _family = None

    def __init__(self, penalty="l2", dual=False, tol=1e-4, C=1.0, fit_intercept=True, intercept_scaling=1.0,
                 class_weight=None, random_state=None, solver="admm", multiclass="ovr", verbose=0, warm_start=False,
                 n_jobs=1, max_iter=100, solver_kwargs=None):
        self.penalty = penalty
        self.dual = dual
        self.tol = tol
        self.C = C
        self.fit_intercept = fit_intercept
        self.intercept_scaling = intercept_scaling
        self.class_weight = class_weight
        self.random_state = random_state
        self.solver = solver
        self.multiclass = multiclass
        self.verbose = verbose
        self.warm_start = warm_start
        self.n_jobs = n_jobs
        self.max_iter = max_iter
        self.solver_kwargs = solver_kwargs

    def _get_solver_kwargs(self):
        """glm.py:135-167: the unregularised solvers drop the regulariser; ``solver_kwargs`` overrides.  As in the
        reference, a ``lamduh`` / ``regularizer`` that ``solver_kwargs`` hands to 'newton' or 'gradient_descent' reaches
        the solver and is ignored there (their functions take no regulariser)."""
        kw = {"max_iter": self.max_iter, "tol": self.tol, "regularizer": self.penalty, "lamduh": 1 / self.C}
        if self.solver in ("gradient_descent", "newton"):
            kw.pop("regularizer")
            kw.pop("lamduh")
        if self.solver_kwargs:
            kw.update(self.solver_kwargs)
        if self.solver not in _SOLVERS:
            raise ValueError("'solver' must be {}. Got '{}' instead".format(_SOLVERS, self.solver))
        return kw

    def fit(self, X, y=None):
        """Fit the model on the training data.  X: every input KMeans takes (``host_resident`` included), or sparse X
        (a ChunkedArray of torch sparse CSR blocks, a torch CSR tensor, a scipy.sparse matrix); y: numpy, torch,
        ``ChunkedArray`` or dask, chunked any way."""
        kw = self._get_solver_kwargs()
        Xs = _sparse_data(X)
        X = Xs if Xs is not None else _device_data(X)
        ys = _y_chunks(y, X, type(self).__name__ + ".fit")
        solver = _SOLVER_FNS[self.solver]
        if Xs is None:
            P = _Passes(X, ys, self._family, self.fit_intercept)
        else:
            P = _SparsePasses(X, ys, self._family, self.fit_intercept)
            if P.p > SPARSE_NEWTON_MAX_P:
                if self.solver == "newton":
                    raise ValueError("solver='newton' needs the (p, p) Hessian, which is too large for sparse input "
                                     "with p = %d > %d coefficients; use 'lbfgs', 'gradient_descent' or "
                                     "'proximal_grad'" % (P.p, SPARSE_NEWTON_MAX_P))
                if self.solver == "admm" and kw.get("regularizer") != "l1":
                    solver = lbfgs                   # the same l2 objective without the Hessian (pgtol = tol)
        self._coef = np.asarray(solver(P, **kw), dtype=np.float64)
        if self.fit_intercept:
            self.coef_ = self._coef[:-1]
            self.intercept_ = float(self._coef[-1])
        else:
            self.coef_ = self._coef
        return self

    # -- predict ---------------------------------------------------------------------------------------------------
    def _pass(self, X, mode):
        """One predict pass: mu per row (float64) or mu > 0.5 (bool), as device-resident ChunkedArray blocks."""
        if getattr(self, "_coef", None) is None:
            raise NotFittedError("This %s instance is not fitted yet. Call 'fit' with appropriate arguments before "
                                 "using this estimator." % type(self).__name__)
        Xs = _sparse_data(X)
        X = Xs if Xs is not None else _device_data(X)
        be, d = X.backend, X.d
        if d != len(self.coef_):
            raise ValueError("X has %d features, but %s is expecting %d features as input"
                             % (d, type(self).__name__, len(self.coef_)))
        beta = np.zeros(d + 1)
        beta[: len(self._coef)] = self._coef
        bd = torch.as_tensor(beta).to(be.device)
        outs = []
        for x in (X.blocks if Xs is not None else X.chunks):
            n = int(x[3]) if Xs is not None else int(x.shape[0])
            o = be.empty((n,), torch.float64 if mode == _PREDICT else torch.uint8)
            if Xs is not None:
                be.glm_csr_pass_chunk(x, d, None, bd, self._family, mode, out=o)
            else:
                be.glm_pass_chunk(x, None, bd, self._family, mode, out=o)
            outs.append(o if mode == _PREDICT else o.view(torch.bool))
        return X, outs

    def _global_mean(self, X, y, outs, term):
        """sum_i term(y_i, out_i) / n over every rank: one all-reduce of [sum, n]."""
        ys = _y_chunks(y, X, type(self).__name__ + ".score")
        red = torch.zeros(2, dtype=torch.float64, device=X.backend.device)
        for yy, o in zip(ys, outs):
            red[0] += term(yy, o).sum(dtype=torch.float64)
        red[1] = float(X.n_local)
        X.comm.allreduce_sum_(red)
        s, n = red.cpu().numpy()
        return s, n


class LogisticRegression(_GLM):
    """Logistic regression (API of dask_ml.linear_model.LogisticRegression, glm.py:200-263).

    Attributes: ``coef_`` (n_features,) float64; ``intercept_`` float (only with ``fit_intercept``)."""

    _family = LOGISTIC

    def predict(self, X):
        """``predict_proba(X) > 0.5``: a bool ChunkedArray on the device, as the reference returns."""
        _, outs = self._pass(X, _LABEL)
        return ChunkedArray(outs)

    def predict_proba(self, X):
        """The (n,) float64 probability of class 1, sigmoid(X beta): a device-resident ChunkedArray."""
        _, outs = self._pass(X, _PREDICT)
        return ChunkedArray(outs)

    def score(self, X, y):
        """The mean accuracy of ``predict(X)`` against y."""
        X, outs = self._pass(X, _LABEL)
        s, n = self._global_mean(X, y, outs, lambda yy, o: (yy == o.to(torch.float64)).to(torch.float64))
        return float(s / n)


class LinearRegression(_GLM):
    """Least squares (API of dask_ml.linear_model.LinearRegression, glm.py:266-324)."""

    _family = NORMAL

    def predict(self, X):
        """X beta: a float64 device-resident ChunkedArray."""
        _, outs = self._pass(X, _PREDICT)
        return ChunkedArray(outs)

    def score(self, X, y):
        """The mean squared error of ``predict(X)``.  The reference's docstring promises R^2, but it returns
        ``mean_squared_error(y, self.predict(X))`` (glm.py:300-324), and so does this method."""
        X, outs = self._pass(X, _PREDICT)
        s, n = self._global_mean(X, y, outs, lambda yy, o: (yy - o) ** 2)
        return float(s / n)


class PoissonRegression(_GLM):
    """Poisson regression (API of dask_ml.linear_model.PoissonRegression, glm.py:327-362)."""

    _family = POISSON

    def predict(self, X):
        """exp(X beta): a float64 device-resident ChunkedArray."""
        _, outs = self._pass(X, _PREDICT)
        return ChunkedArray(outs)

    def get_deviance(self, X, y):
        """2 sum_i (y_i log(y_i / mu_i) - (y_i - mu_i)), with 0 log 0 = 0."""
        X, outs = self._pass(X, _PREDICT)
        s, _ = self._global_mean(X, y, outs, lambda yy, mu: 2.0 * (torch.special.xlogy(yy, yy / mu) - (yy - mu)))
        return float(s)
