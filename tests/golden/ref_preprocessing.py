"""TEST INFRASTRUCTURE — run the UNMODIFIED reference ``dask_ml/preprocessing/data.py`` without dask.

    BKM_REFERENCE=<dask-ml checkout> python tests/golden/ref_preprocessing.py   # regenerates tests/golden/ref_pp_*.npz

``ref_shim.install()`` provides the eager stand-in for the slice of dask the KMeans path uses.  The scalers need a few
more pieces, added here:
  * ``Array.mean``, ``var``, ``max``, ``copy``, ``__eq__``, boolean ``__setitem__``, ``__rtruediv__``, ``__rsub__``,
    and numpy scalars deferring to the stand-in;
  * ``da.sqrt`` on the stand-in, ``da.vstack`` stacking rows, ``dask.compute``;
  * ``da.percentile`` as ``np.percentile`` over the whole column: the shim's stand-in for dask's per-chunk merge;
  * ``sklearn.preprocessing.data`` as an alias of ``sklearn.preprocessing._data``, and ``distutils.version`` (gone
    from Python 3.12) with a ``LooseVersion`` built on ``packaging``;
  * the module's ``check_is_fitted`` taking several attribute names positionally, as scikit-learn < 0.22 did.
Each case records the fitted attributes, ``transform`` of X and ``inverse_transform`` of that output.  The reference
file is then loaded with importlib, byte for byte.  tests/test_preprocessing_host.py and
tests/test_gpu_preprocessing.py replay the fixtures; neither needs the reference checkout.
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

ATTRS = {"StandardScaler": ("mean_", "var_", "scale_", "n_samples_seen_"),
         "MinMaxScaler": ("data_min_", "data_max_", "data_range_", "scale_", "min_", "n_samples_seen_"),
         "RobustScaler": ("center_", "scale_")}


def install():
    ref = ref_shim.install()
    da, Array = ref.da, ref.da.Array
    Array.__array_ufunc__ = None

    def full(x):
        return x.compute() if isinstance(x, Array) else x

    Array.__eq__ = lambda self, o: self._bin(o, np.equal)
    Array.__hash__ = object.__hash__
    Array.__rsub__ = lambda self, o: self._bin(o, lambda a, b: b - a)
    Array.__rtruediv__ = lambda self, o: self._bin(o, lambda a, b: b / a)
    Array.max = lambda self, axis=None: self._like(self.compute().max(axis=axis))
    Array.mean = lambda self, axis=None: Array([np.asarray(self.compute().mean(axis=axis))])
    Array.var = lambda self, axis=None, ddof=0: Array([np.asarray(self.compute().var(axis=axis, ddof=ddof))])
    Array.copy = lambda self: Array([b.copy() for b in self.blocks])

    def setitem(self, key, value):
        a = self.compute().copy()
        a[full(key)] = value
        self.blocks = [a]

    Array.__setitem__ = setitem
    da.sqrt = ref_shim._elementwise(np.sqrt)
    da.vstack = lambda arrs: Array([np.vstack([full(a) for a in arrs])])
    da.percentile = lambda a, q: Array([np.asarray(np.percentile(full(a), q))])
    sys.modules["dask"].compute = ref_shim._compute

    import sklearn.preprocessing
    import sklearn.preprocessing._data as skdata

    sys.modules["sklearn.preprocessing.data"] = skdata
    sklearn.preprocessing.data = skdata
    try:
        import distutils.version  # noqa: F401
    except ImportError:
        from packaging.version import Version

        dv = types.ModuleType("distutils.version")

        class LooseVersion(object):
            def __init__(self, v):
                self.v = Version(str(v).split("+")[0])

            def __ge__(self, o):
                return self.v >= Version(str(o))

        dv.LooseVersion = LooseVersion
        dist = types.ModuleType("distutils")
        dist.version = dv
        sys.modules["distutils"] = dist
        sys.modules["distutils.version"] = dv

    root = os.path.join(ref_shim.REF, "dask_ml")
    pkg = types.ModuleType("dask_ml.preprocessing")
    pkg.__path__ = [os.path.join(root, "preprocessing")]
    sys.modules["dask_ml.preprocessing"] = pkg
    path = os.path.join(root, "preprocessing", "data.py")
    spec = importlib.util.spec_from_file_location("dask_ml.preprocessing.data", path)
    m = importlib.util.module_from_spec(spec)
    sys.modules["dask_ml.preprocessing.data"] = m
    spec.loader.exec_module(m)
    from sklearn.utils.validation import check_is_fitted

    # RobustScaler.inverse_transform passes two attribute names positionally (scikit-learn < 0.22's signature)
    m.check_is_fitted = lambda est, attributes=None, *more: check_is_fitted(est, [attributes, *more])
    return ref, m


def data(case):
    rng = np.random.RandomState(case["seed"])
    n, d = case["n"], case["d"]
    kind = case.get("kind", "normal")
    if kind == "offset":
        X = 1e6 + rng.standard_normal((n, d))
    elif kind == "integers":
        X = rng.randint(0, 5, size=(n, d)).astype(np.float64)        # many duplicates
    else:
        X = rng.standard_normal((n, d)) * rng.uniform(0.5, 3.0, d) + rng.uniform(-5, 5, d)
    for j in case.get("constant", []):
        X[:, j] = 2.5
    for j in case.get("nan", []):
        X[rng.randint(0, n, size=3), j] = np.nan
    return X.astype(case["dtype"])


CASES = {
    "ref_pp_std_f64_offset": dict(cls="StandardScaler", n=1500, d=4, seed=1, dtype="float64", chunks=400,
                                  kind="offset"),
    "ref_pp_std_f32": dict(cls="StandardScaler", n=1200, d=5, seed=2, dtype="float32", chunks=500),
    "ref_pp_std_nomean": dict(cls="StandardScaler", n=900, d=3, seed=3, dtype="float64", chunks=300,
                              params=dict(with_mean=False)),
    "ref_pp_std_nostd": dict(cls="StandardScaler", n=900, d=3, seed=4, dtype="float64", chunks=300,
                             params=dict(with_std=False)),
    "ref_pp_std_neither": dict(cls="StandardScaler", n=700, d=3, seed=5, dtype="float32", chunks=300,
                               params=dict(with_mean=False, with_std=False)),
    "ref_pp_std_const": dict(cls="StandardScaler", n=800, d=4, seed=6, dtype="float64", chunks=300, constant=[1]),
    "ref_pp_std_nan": dict(cls="StandardScaler", n=800, d=4, seed=7, dtype="float64", chunks=300, nan=[2]),
    "ref_pp_mm_default": dict(cls="MinMaxScaler", n=1000, d=5, seed=8, dtype="float64", chunks=300),
    "ref_pp_mm_f32_range": dict(cls="MinMaxScaler", n=1000, d=5, seed=9, dtype="float32", chunks=400,
                                params=dict(feature_range=(-1, 3))),
    "ref_pp_mm_const": dict(cls="MinMaxScaler", n=600, d=3, seed=10, dtype="float64", chunks=250, constant=[0]),
    "ref_pp_rob_default": dict(cls="RobustScaler", n=1001, d=5, seed=11, dtype="float64", chunks=300),
    "ref_pp_rob_f32_10_90": dict(cls="RobustScaler", n=1200, d=4, seed=12, dtype="float32", chunks=500,
                                 params=dict(quantile_range=(10, 90))),
    "ref_pp_rob_0_100": dict(cls="RobustScaler", n=777, d=3, seed=13, dtype="float64", chunks=300,
                             params=dict(quantile_range=(0, 100))),
    "ref_pp_rob_50_50": dict(cls="RobustScaler", n=640, d=3, seed=14, dtype="float64", chunks=300,
                             params=dict(quantile_range=(50, 50))),
    "ref_pp_rob_dups": dict(cls="RobustScaler", n=900, d=4, seed=15, dtype="float64", chunks=350, kind="integers"),
}

ERRORS = {
    "MinMaxScaler": dict(feature_range=(2, 2)),
    "RobustScaler": dict(quantile_range=(80, 20)),
}


def main():
    ref, pp = install()
    da = ref.da
    manifest = {"reference": "mrocklin/dask-ml @ 0310a90 preprocessing/data.py run through "
                             "tests/golden/ref_preprocessing.py", "cases": {}, "errors": {}}
    for name, case in CASES.items():
        X = data(case)
        rows = case["chunks"]
        est = getattr(pp, case["cls"])(**case.get("params", {}))
        with np.errstate(all="ignore"):
            est.fit(da.from_array(X, chunks=(rows, X.shape[1])))               # the reference's own fit
            t = est.transform(da.from_array(X, chunks=(rows, X.shape[1])))
            t = np.asarray(t.compute() if hasattr(t, "compute") else t)
            inv = est.inverse_transform(da.from_array(t, chunks=(rows, X.shape[1])))
            inv = np.asarray(inv.compute() if hasattr(inv, "compute") else inv)
        out = dict(X=X, chunks=rows, transform=t, inverse_transform=inv)
        dtypes = {}
        for a in ATTRS[case["cls"]]:
            if hasattr(est, a):
                v = getattr(est, a)
                out["attr_" + a] = np.asarray(v)
                dtypes[a] = str(np.asarray(v).dtype)
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
        manifest["cases"][name] = dict(case, attr_dtypes=dtypes, transform_dtype=str(t.dtype),
                                       inverse_dtype=str(inv.dtype))
        print(name, manifest["cases"][name], flush=True)
    for cls, params in ERRORS.items():
        try:
            getattr(pp, cls)(**params).fit(da.from_array(np.ones((10, 2)), chunks=(5, 2)))
            manifest["errors"][cls] = None
        except Exception as e:
            manifest["errors"][cls] = dict(params={k: list(v) for k, v in params.items()}, type=type(e).__name__,
                                           message=str(e))
    with open(os.path.join(HERE, "REF_PREPROCESSING_MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1)


if __name__ == "__main__":
    main()
