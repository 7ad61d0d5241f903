"""TEST INFRASTRUCTURE — run the UNMODIFIED reference ``dask_ml/naive_bayes.py`` without dask.

    BKM_REFERENCE=<dask-ml checkout> python tests/golden/ref_naive_bayes.py   # regenerates tests/golden/ref_nb_*.npz

``ref_shim.install()`` provides the eager stand-in for the slice of dask the KMeans path uses.  GaussianNB needs a few
more pieces, added here:
  * ``Array.__eq__``, boolean ``__getitem__`` (``X[y == c]``), ``max``, ``reshape``, ``__neg__``, ``mean``, ``var``,
    and numpy scalars deferring to the stand-in;
  * ``da.exp``, ``da.log``, ``da.sum``, ``da.stack``, ``da.argmax``;
  * ``dask.delayed`` of a plain value (``delayed(self.classes_)[labels]`` in ``predict``);
  * a stub ``dask_ml._partial`` whose mixin is a class, because the module defines PartialMultinomialNB and
    PartialBernoulliNB at import.
Each case records the fit on all of X and the three predict methods on X's first 300 rows (150-row chunks).
The reference file is then loaded with importlib, byte for byte.  tests/test_naive_bayes_host.py and
tests/test_gpu_naive_bayes.py replay the fixtures; neither needs the reference checkout.
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import ref_shim  # noqa: E402


def install():
    ref = ref_shim.install()
    da, Array = ref.da, ref.da.Array
    Array.__array_ufunc__ = None

    def full(x):
        return x.compute() if isinstance(x, Array) else x

    getitem = Array.__getitem__
    Array.__getitem__ = lambda self, key: getitem(self, full(key))
    Array.__eq__ = lambda self, o: self._bin(o, np.equal)
    Array.__hash__ = object.__hash__
    Array.__neg__ = lambda self: self._like(-self.compute())
    Array.__rsub__ = lambda self, o: self._bin(o, lambda a, b: b - a)
    Array.max = lambda self, axis=None: self._like(self.compute().max(axis=axis))
    Array.reshape = lambda self, *shape: self._like(self.compute().reshape(*shape))
    Array.mean = lambda self, axis=None: Array([np.asarray(self.compute().mean(axis=axis))])
    Array.var = lambda self, axis=None, ddof=0: Array([np.asarray(self.compute().var(axis=axis, ddof=ddof))])

    da.exp = ref_shim._elementwise(np.exp)
    da.log = ref_shim._elementwise(np.log)
    da.sum = lambda x, axis=None: x._like(full(x).sum(axis=axis)) if isinstance(x, Array) else np.sum(x, axis=axis)
    da.stack = lambda arrs: Array([np.stack([full(a) for a in arrs])])
    da.argmax = lambda x, axis=None: x._like(np.argmax(full(x), axis=axis))

    class _Value(object):
        """dask.delayed of a plain value: indexing it indexes the value."""

        def __init__(self, v):
            self.v = v

        def __getitem__(self, key):
            return Array([np.asarray(self.v)[full(key)]])

    wrap = ref_shim._delayed

    def delayed(obj=None, **kw):
        return wrap(obj, **kw) if callable(obj) else _Value(obj)

    sys.modules["dask"].delayed = delayed

    partial = types.ModuleType("dask_ml._partial")

    class _BigPartialFitMixin(object):
        pass

    partial._BigPartialFitMixin = _BigPartialFitMixin
    partial._copy_partial_doc = lambda cls: cls
    sys.modules["dask_ml._partial"] = partial

    path = os.path.join(ref_shim.REF, "dask_ml", "naive_bayes.py")
    spec = importlib.util.spec_from_file_location("dask_ml.naive_bayes", path)
    m = importlib.util.module_from_spec(spec)
    sys.modules["dask_ml.naive_bayes"] = m
    spec.loader.exec_module(m)
    return ref, m


def data(case):
    """(X, y) of a case: K Gaussian classes with per-class means and scales."""
    rng = np.random.RandomState(case["seed"])
    n, d, K = case["n"], case["d"], case["K"]
    means = rng.uniform(-3, 3, size=(K, d)) + case.get("offset", 0.0)
    scales = rng.uniform(0.5, 2.0, size=(K, d))
    y = rng.randint(0, K, size=n).astype(np.int64)
    X = means[y] + scales[y] * rng.standard_normal((n, d))
    for c, r in case.get("singleton", []):          # class c reduced to the one row r
        y[(y == c) & (np.arange(n) != r)] = (c + 1) % K
        y[r] = c
    for c, j in case.get("constant", []):            # feature j constant within class c
        X[y == c, j] = means[c, j]
    return X.astype(case["dtype"]), y


PREDICT_ROWS, PREDICT_CHUNKS = 300, 150     # predict on the first rows only: (n, K) float64 outputs do not compress

CASES = {
    "ref_nb_f64_k3": dict(n=1500, d=6, K=3, seed=1, dtype="float64", chunks=400),
    "ref_nb_f32_k4": dict(n=1200, d=5, K=4, seed=2, dtype="float32", chunks=500),
    "ref_nb_f64_offset": dict(n=1600, d=4, K=3, seed=3, dtype="float64", chunks=700, offset=1e4),
    "ref_nb_f64_k40": dict(n=2000, d=8, K=40, seed=4, dtype="float64", chunks=1500),
    # label 2 is not modelled (its rows enter no sum but count in n); class 9 has no rows; classes_ keeps this order
    "ref_nb_f64_classes": dict(n=1000, d=3, K=4, seed=5, dtype="float64", chunks=300, classes=[3, 0, 1, 9]),
    # class 1 is a single row and class 2 has a constant feature: both have a zero variance, hence NaN likelihoods
    "ref_nb_f64_nan_classes": dict(n=800, d=3, K=4, seed=6, dtype="float64", chunks=300, singleton=[(1, 17)],
                                   constant=[(2, 1)]),
}


def main():
    ref, nb = install()
    da = ref.da
    manifest = {"reference": "mrocklin/dask-ml @ 0310a90 naive_bayes.py run through tests/golden/ref_naive_bayes.py",
                "cases": {}}
    for name, case in CASES.items():
        X, y = data(case)
        rows = case["chunks"]
        Xd = da.from_array(X, chunks=(rows, X.shape[1]))
        yd = da.from_array(y, chunks=rows)
        Xp = da.from_array(X[:PREDICT_ROWS], chunks=(PREDICT_CHUNKS, X.shape[1]))
        with np.errstate(all="ignore"):
            est = nb.GaussianNB(classes=case.get("classes")).fit(Xd, yd)     # the reference's own fit
            out = dict(X=X, y=y, chunks=rows, predict_chunks=PREDICT_CHUNKS, classes_=np.asarray(est.classes_),
                       theta=np.asarray(est.theta_.compute()), sigma=np.asarray(est.sigma_.compute()),
                       class_count=np.asarray(est.class_count_.compute()),
                       class_prior=np.asarray(est.class_prior_.compute()),
                       predict=np.asarray(est.predict(Xp).compute()),
                       predict_proba=np.asarray(est.predict_proba(Xp).compute()),
                       predict_log_proba=np.asarray(est.predict_log_proba(Xp).compute()))
        if case.get("classes") is not None:
            out["classes"] = np.asarray(case["classes"])
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
        lp = out["predict_log_proba"]
        manifest["cases"][name] = dict(
            {k: v for k, v in case.items()}, predict_rows=int(len(out["predict"])), theta_dtype=str(out["theta"].dtype),
            classes_=[int(c) for c in out["classes_"]], class_count=[float(c) for c in out["class_count"]],
            class_prior_sum=float(out["class_prior"].sum()),
            nan_theta_classes=[int(i) for i in np.nonzero(np.isnan(out["theta"]).any(1))[0]],
            predict_counts={str(int(c)): int((out["predict"] == c).sum()) for c in np.unique(out["predict"])},
            nan_log_proba_rows=int(np.isnan(lp).any(1).sum()),
            finite_log_proba_sum=float(lp[np.isfinite(lp)].sum()))
        print(name, manifest["cases"][name], flush=True)
    with open(os.path.join(HERE, "REF_NAIVE_BAYES_MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1)


if __name__ == "__main__":
    main()
