"""TEST INFRASTRUCTURE — run the UNMODIFIED reference ``SimpleImputer`` (dask_ml/impute.py) without dask.

    BKM_REFERENCE=<dask-ml checkout> python tests/golden/ref_impute.py   # regenerates tests/golden/ref_imp_*.npz

Built on ``ref_preprocessing.install()`` (itself on ``ref_shim``).  The imputer needs a few more pieces, added here:
  * ``da.nanmean`` over a whole axis of the stand-in, ``da.isnull`` and a three-argument ``da.where`` (the shim's
    ``where`` is the one-argument form the KMeans path uses);
  * ``dask.dataframe.Series`` / ``DataFrame`` stand-ins that are not pandas' types, so that numpy input takes the
    reference's numpy branch and the stand-in array its array branch (the reference's type tuple is built from them);
  * an adapter for ``check_array(force_all_finite=...)``, which scikit-learn 1.9 spells ``ensure_all_finite``.
The reference file is then loaded with importlib, byte for byte.  Cases:
  * its array path (``da.Array`` input): ``mean`` and ``constant``, NaN missing values, ``statistics_`` and
    ``da.where(da.isnull(X), statistics_, X)``;
  * its numpy path (which hands the work to scikit-learn): all four strategies, NaN and numeric missing values, an
    all-missing column, ``keep_empty_features``, ``add_indicator`` with ``inverse_transform``;
  * the three error cases of its tests/test_impute.py on the array path.  The third (``median`` on a dask array) is
    the restriction this package lifts: its manifest entry carries ``expected_difference``.
tests/test_impute_host.py and tests/test_gpu_impute.py replay the fixtures; neither needs the reference checkout.
"""
import importlib.util
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
    ref, _ = ref_preprocessing.install()
    da, Array = ref.da, ref.da.Array

    def full(x):
        return x.compute() if isinstance(x, Array) else np.asarray(x)

    def nanmean(a, axis=None):
        with np.errstate(all="ignore"), warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            return Array([np.asarray(np.nanmean(full(a), axis=axis))])

    shim_where = da.where

    def where(cond, *ab):
        if not ab:
            return shim_where(cond)
        return Array([np.where(full(cond), full(ab[0]), full(ab[1]))])

    da.nanmean = nanmean
    da.isnull = ref_shim._elementwise(np.isnan)
    da.where = where

    import sklearn.utils.validation as skv

    sk_check = skv.check_array

    def check_array(array, *a, **k):
        if "force_all_finite" in k:
            k["ensure_all_finite"] = k.pop("force_all_finite")
        return sk_check(array, *a, **k)

    ref.utils.sk_validation = type("V", (), {"check_array": staticmethod(check_array)})
    path = os.path.join(ref_shim.REF, "dask_ml", "impute.py")
    spec = importlib.util.spec_from_file_location("dask_ml.impute", path)
    m = importlib.util.module_from_spec(spec)
    sys.modules["dask_ml.impute"] = m
    spec.loader.exec_module(m)
    return ref, m


def data(case):
    rng = np.random.RandomState(case["seed"])
    n, d = case["n"], case["d"]
    X = rng.standard_normal((n, d)) * 3 + 10
    X[:, 1] = rng.randint(0, 5, n)                                   # categorical: a real mode
    if d > 2:
        X[:, 2] = np.round(rng.standard_normal(n), 1)                 # duplicates and ties
    miss = np.nan if case.get("missing", "nan") == "nan" else case["missing"]
    X[rng.uniform(size=(n, d)) < 0.2] = miss
    for j in case.get("empty", []):
        X[:, j] = miss
    return X.astype(case["dtype"]), miss


CASES = {
    "ref_imp_array_mean": dict(path="array", n=400, d=4, seed=1, dtype="float64", chunks=150),
    "ref_imp_array_constant": dict(path="array", n=400, d=4, seed=2, dtype="float64", chunks=150,
                                   params=dict(strategy="constant", fill_value=-999.0)),
    "ref_imp_np_mean_f32": dict(path="numpy", n=500, d=4, seed=3, dtype="float32", chunks=200),
    "ref_imp_np_median": dict(path="numpy", n=501, d=4, seed=4, dtype="float64", chunks=200,
                              params=dict(strategy="median")),
    "ref_imp_np_most_frequent": dict(path="numpy", n=500, d=4, seed=5, dtype="float64", chunks=200,
                                     params=dict(strategy="most_frequent")),
    "ref_imp_np_constant": dict(path="numpy", n=300, d=3, seed=6, dtype="float32", chunks=100,
                                params=dict(strategy="constant", fill_value=7)),
    "ref_imp_np_numeric_missing": dict(path="numpy", n=400, d=4, seed=7, dtype="float64", chunks=150, missing=-1.0,
                                       params=dict(strategy="median", missing_values=-1.0)),
    "ref_imp_np_empty_column": dict(path="numpy", n=300, d=4, seed=8, dtype="float64", chunks=100, empty=[3],
                                    params=dict(strategy="most_frequent", add_indicator=True)),
    "ref_imp_np_keep_empty": dict(path="numpy", n=300, d=4, seed=9, dtype="float64", chunks=100, empty=[0],
                                  params=dict(strategy="mean", keep_empty_features=True)),
    "ref_imp_np_indicator": dict(path="numpy", n=400, d=4, seed=10, dtype="float32", chunks=150, missing=0.0,
                                 params=dict(strategy="median", missing_values=0.0, add_indicator=True)),
}

ERRORS = {
    "strategy_other": dict(strategy="other"),
    "missing_values_foo": dict(missing_values="foo"),
    "array_median": dict(strategy="median"),
}
EXPECTED_DIFFERENCE = {"array_median": "dask_ml_b200 runs every strategy on every input kind; the reference's array "
                                       "path allows only mean and constant"}


def main():
    ref, imp = install()
    da = ref.da
    manifest = {"reference": "mrocklin/dask-ml @ 0310a90 impute.py run through tests/golden/ref_impute.py",
                "cases": {}, "errors": {}}
    for name, case in CASES.items():
        X, miss = data(case)
        rows = case["chunks"]
        est = imp.SimpleImputer(**case.get("params", {}))
        src = da.from_array(X, chunks=(rows, X.shape[1])) if case["path"] == "array" else X
        with np.errstate(all="ignore"), warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            est.fit(src)
            t = est.transform(src)
            t = np.asarray(t.compute() if hasattr(t, "compute") else t)
        out = dict(X=X, chunks=rows, statistics_=np.asarray(est.statistics_, dtype=np.float64), transform=t)
        if case.get("params", {}).get("add_indicator"):
            out["inverse"] = np.asarray(est.inverse_transform(t))
            out["features_"] = np.asarray(est.indicator_.features_)
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
        manifest["cases"][name] = dict(
            case, missing="nan" if np.isnan(miss) else float(miss), statistics_dtype=str(np.asarray(est.statistics_).dtype),
            transform_dtype=str(t.dtype), warnings=[str(w.message) for w in caught if "Skipping" in str(w.message)])
        print(name, manifest["cases"][name], flush=True)
    X = np.random.RandomState(0).uniform(size=(10, 4))
    X[X < 0.5] = np.nan                                             # the reference's tests/test_impute.py data
    for key, params in ERRORS.items():
        try:
            imp.SimpleImputer(**params).fit(da.from_array(X, chunks=(5, 4)))
            manifest["errors"][key] = None
        except Exception as e:
            manifest["errors"][key] = dict(params=params, type=type(e).__name__, message=str(e))
        if key in EXPECTED_DIFFERENCE:
            manifest["errors"][key]["expected_difference"] = EXPECTED_DIFFERENCE[key]
    with open(os.path.join(HERE, "REF_IMPUTE_MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1)


if __name__ == "__main__":
    main()
