"""TEST INFRASTRUCTURE — run the UNMODIFIED reference ``QuantileTransformer`` (dask_ml/preprocessing/data.py) without
dask.

    BKM_REFERENCE=<dask-ml checkout> python tests/golden/ref_quantile.py   # regenerates tests/golden/ref_qt_*.npz

Built on ``ref_preprocessing.install()``, which loads the reference file byte for byte.  QuantileTransformer needs a
few more pieces, added here:
  * ``Array.__neg__`` and ``da.clip`` on the stand-in;
  * adapters between the reference's ``_check_inputs(X, accept_sparse_negative)`` (scikit-learn 0.20's signature) and
    the installed scikit-learn's ``_check_inputs(X, in_fit, accept_sparse_negative, copy)``, in both directions:
    scikit-learn's ``fit`` / ``transform`` call the reference's method with the new arguments, and the reference's
    ``super()._check_inputs`` call reaches scikit-learn's method without ``in_fit``, which is taken from the outer call;
  * the inverse through the reference's own ``_transform(X, inverse=True)``: scikit-learn's ``inverse_transform``
    converts the stand-in to numpy first, which the reference never sees.
Each case records ``n_quantiles_``, ``references_``, ``quantiles_``, the transform of X and of a second array Y that
reaches beyond the fitted range, and the inverse of both outputs.  The manifest is separate from
REF_PREPROCESSING_MANIFEST.json, whose cases the scaler replay reads.  tests/test_quantile_host.py and
tests/test_gpu_quantile.py replay the fixtures; neither needs the reference checkout.
"""
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import ref_preprocessing  # noqa: E402
import ref_shim  # noqa: E402


def install():
    ref, m = ref_preprocessing.install()
    da, Array = ref.da, ref.da.Array
    Array.__neg__ = lambda self: Array([-b for b in self.blocks])
    da.clip = ref_shim._elementwise(np.clip)

    import sklearn.preprocessing._data as skdata

    ref_check = m.QuantileTransformer._check_inputs
    sk_check = skdata.QuantileTransformer._check_inputs
    outer = {"in_fit": True}

    def check_new_to_ref(self, X, in_fit=True, accept_sparse_negative=False, copy=False):
        outer["in_fit"] = in_fit
        return ref_check(self, X, accept_sparse_negative=accept_sparse_negative)

    def check_ref_to_new(self, X, in_fit=None, accept_sparse_negative=False, copy=False):
        return sk_check(self, X, outer["in_fit"] if in_fit is None else in_fit, accept_sparse_negative, copy)

    m.QuantileTransformer._check_inputs = check_new_to_ref
    skdata.QuantileTransformer._check_inputs = check_ref_to_new
    return ref, m


def data(case, seed_offset=0, spread=1.0):
    """X of a case (and, with seed_offset / spread, the second array Y that reaches beyond X's range)."""
    rng = np.random.RandomState(case["seed"] + seed_offset)
    n, d = case["n"], case["d"]
    X = rng.standard_normal((n, d)) * rng.uniform(0.5, 3.0, d) + rng.uniform(-5, 5, d)
    if case.get("kind") == "offset":
        X = 1e6 + rng.standard_normal((n, d))
    X = X * spread
    for j in case.get("integers", []):
        X[:, j] = rng.randint(0, 8, n)                             # repeated quantiles
    for j in case.get("constant", []):
        X[:, j] = 2.5
    for j in case.get("nan", []):
        X[rng.randint(0, n), j] = np.nan
    for j in case.get("inf", []):
        X[rng.randint(0, n, 3), j] = np.inf
        X[rng.randint(0, n, 2), j] = -np.inf
    return X.astype(case["dtype"])


CASES = {
    "ref_qt_f64_default": dict(n=1500, d=3, seed=1, dtype="float64", chunks=400),
    "ref_qt_f64_normal": dict(n=1500, d=3, seed=2, dtype="float64", chunks=400,
                              params=dict(output_distribution="normal")),
    "ref_qt_f32_integers": dict(n=1200, d=3, seed=3, dtype="float32", chunks=500, integers=[1],
                                params=dict(n_quantiles=200)),
    "ref_qt_f32_integers_normal": dict(n=1200, d=3, seed=4, dtype="float32", chunks=500, integers=[0],
                                       params=dict(n_quantiles=200, output_distribution="normal")),
    "ref_qt_offset": dict(n=1100, d=2, seed=5, dtype="float64", chunks=300, kind="offset"),
    "ref_qt_small_nq": dict(n=800, d=3, seed=6, dtype="float64", chunks=300, params=dict(n_quantiles=10)),
    "ref_qt_n_below_nq": dict(n=300, d=3, seed=7, dtype="float64", chunks=128),
    "ref_qt_n1": dict(n=1, d=3, seed=8, dtype="float64", chunks=1),
    "ref_qt_nan": dict(n=600, d=3, seed=9, dtype="float64", chunks=250, nan=[1], params=dict(n_quantiles=100)),
    "ref_qt_inf": dict(n=600, d=3, seed=10, dtype="float64", chunks=250, inf=[2],
                       params=dict(n_quantiles=100, output_distribution="normal")),
    "ref_qt_constant": dict(n=500, d=3, seed=11, dtype="float32", chunks=200, constant=[0],
                            params=dict(n_quantiles=50)),
}

ERRORS = {
    "n_quantiles_above_subsample": dict(n_quantiles=2000, subsample=1000),
    "n_quantiles_zero": dict(n_quantiles=0),
    "distribution": dict(output_distribution="gamma"),
}


def main():
    ref, pp = install()
    da = ref.da
    manifest = {"reference": "mrocklin/dask-ml @ 0310a90 preprocessing/data.py QuantileTransformer run through "
                             "tests/golden/ref_quantile.py", "cases": {}, "errors": {}}
    for name, case in CASES.items():
        X = data(case)
        Y = data(case, seed_offset=1000, spread=1.5)
        rows = case["chunks"]
        est = pp.QuantileTransformer(**case.get("params", {}))
        with np.errstate(all="ignore"), warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            est.fit(da.from_array(X, chunks=(rows, X.shape[1])))         # the reference's own fit
            tx = np.asarray(est.transform(da.from_array(X, chunks=(rows, X.shape[1]))).compute())
            ty = np.asarray(est.transform(da.from_array(Y, chunks=(rows, X.shape[1]))).compute())
            ix = np.asarray(est._transform(da.from_array(tx, chunks=(rows, X.shape[1])), inverse=True).compute())
            iy = np.asarray(est._transform(da.from_array(ty, chunks=(rows, X.shape[1])), inverse=True).compute())
        warned = [str(w.message) for w in caught if "n_quantiles" in str(w.message)]
        out = dict(X=X, Y=Y, chunks=rows, n_quantiles_=est.n_quantiles_, references_=est.references_,
                   quantiles_=est.quantiles_, transform_X=tx, transform_Y=ty, inverse_X=ix, inverse_Y=iy)
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
        manifest["cases"][name] = dict(case, n_quantiles_=int(est.n_quantiles_),
                                       quantiles_dtype=str(est.quantiles_.dtype), transform_dtype=str(tx.dtype),
                                       inverse_dtype=str(ix.dtype), warnings=warned)
        print(name, manifest["cases"][name], flush=True)
    for key, params in ERRORS.items():
        try:
            pp.QuantileTransformer(**params).fit(da.from_array(np.ones((10, 2)), chunks=(5, 2)))
            manifest["errors"][key] = None
        except Exception as e:
            manifest["errors"][key] = dict(params=params, type=type(e).__name__, message=str(e))
    with open(os.path.join(HERE, "REF_QUANTILE_MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1)


if __name__ == "__main__":
    main()
