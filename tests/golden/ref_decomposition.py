"""TEST INFRASTRUCTURE — run the UNMODIFIED reference ``dask_ml/decomposition/pca.py`` and ``truncated_svd.py`` without dask.

    BKM_REFERENCE=<dask-ml checkout> python tests/golden/ref_decomposition.py   # regenerates tests/golden/ref_decomp_*.npz

``ref_shim.install()`` provides the eager stand-in for the slice of dask the KMeans path uses (and loads the reference's
own ``dask_ml/utils.py``, whose ``svd_flip`` is scikit-learn's U-based ``svd_flip`` through ``dask.delayed``).  The
decomposition path needs a few more pieces, added here:
  * ``da.linalg.svd``  -> ``numpy.linalg.svd(full_matrices=False)``, U chunked like X;
  * ``Array.mean`` / ``Array.var`` / ``Array.dot``, ``da.log``, ``da.mean``, and numpy scalars deferring to the stand-in;
  * ``sklearn.decomposition.base`` -> ``sklearn.decomposition._base`` (the module was renamed).
The two reference files are then loaded with importlib, byte for byte.  tests/test_decomposition_host.py and
tests/test_gpu_decomposition.py replay the fixtures; neither needs the reference checkout.

'randomized' has no fixture (``svd_compressed`` is a dask algorithm the stand-in does not provide); it is checked
against scikit-learn's exact top-k instead.
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
    Array.__array_ufunc__ = None                                  # np.float64 * Array -> Array.__rmul__

    def full(x):
        return x.compute() if isinstance(x, Array) else np.asarray(x)

    Array.dot = lambda self, o: self._like(np.dot(self.compute(), full(o)))
    Array.mean = lambda self, axis=None: Array([np.asarray(self.compute().mean(axis=axis))])
    Array.var = lambda self, axis=None, ddof=0: Array([np.asarray(self.compute().var(axis=axis, ddof=ddof))])
    Array.__rtruediv__ = lambda self, o: self._bin(o, lambda a, b: b / a)

    def svd(X):
        U, S, V = np.linalg.svd(full(X), full_matrices=False)
        return (X._like(U) if isinstance(X, Array) else Array([U])), Array([S]), Array([V])

    da.linalg = types.SimpleNamespace(svd=svd)
    da.log = ref_shim._elementwise(np.log)
    da.mean = lambda x: Array([np.asarray(full(x).mean())])

    import sklearn.decomposition
    import sklearn.decomposition._base as base

    sys.modules["sklearn.decomposition.base"] = base
    sklearn.decomposition.base = base

    root = os.path.join(ref_shim.REF, "dask_ml", "decomposition")
    pkg = types.ModuleType("dask_ml.decomposition")
    pkg.__path__ = [root]
    sys.modules["dask_ml.decomposition"] = pkg
    mods = {}
    for name in ("pca", "truncated_svd"):
        spec = importlib.util.spec_from_file_location("dask_ml.decomposition." + name, os.path.join(root, name + ".py"))
        m = importlib.util.module_from_spec(spec)
        sys.modules["dask_ml.decomposition." + name] = m
        spec.loader.exec_module(m)
        mods[name] = m
    return ref, mods["pca"], mods["truncated_svd"]


def data(n, d, seed, offset, dtype):
    rng = np.random.RandomState(seed)
    A = rng.standard_normal((d, d)) * np.linspace(3, 0.2, d)[:, None]
    return (rng.standard_normal((n, d)) @ A + offset).astype(dtype)


# name: (estimator, n, d, seed, offset, dtype, chunks, constructor keywords)
CASES = {
    "ref_decomp_pca_f64_full_all": ("pca", 2000, 12, 1, 0.0, "float64", 500, dict(svd_solver="full")),
    "ref_decomp_pca_f64_tsqr_k5": ("pca", 2000, 12, 2, 0.0, "float64", 700, dict(n_components=5, svd_solver="tsqr")),
    "ref_decomp_pca_f64_whiten_k4": ("pca", 1500, 10, 3, 0.0, "float64", 400,
                                     dict(n_components=4, whiten=True, svd_solver="full")),
    "ref_decomp_pca_f64_offset_k3": ("pca", 2000, 8, 4, 1e4, "float64", 600, dict(n_components=3, svd_solver="tsqr")),
    "ref_decomp_pca_f32_full_k6": ("pca", 2000, 16, 5, 0.0, "float32", 500, dict(n_components=6, svd_solver="full")),
    "ref_decomp_pca_f32_whiten_offset_k3": ("pca", 1800, 9, 6, 1e4, "float32", 600,
                                            dict(n_components=3, whiten=True, svd_solver="tsqr")),
    "ref_decomp_tsvd_f64_k4": ("tsvd", 2000, 12, 7, 3.0, "float64", 500, dict(n_components=4, algorithm="tsqr")),
    "ref_decomp_tsvd_f32_k3": ("tsvd", 1600, 10, 8, 1.0, "float32", 400, dict(n_components=3, algorithm="tsqr")),
}

# (estimator, constructor keywords, n, d): the reference's errors on a small float64 X
ERRORS = [
    ("pca", dict(svd_solver="arpack"), 50, 6),
    ("pca", dict(n_components=0.5), 50, 6),
    ("pca", dict(n_components=7, svd_solver="full"), 50, 6),
    ("pca", dict(n_components=7), 50, 6),
    ("pca", dict(n_components=-1, svd_solver="tsqr"), 50, 6),
    ("pca", dict(n_components=700, svd_solver="auto"), 600, 800),
    ("tsvd", dict(n_components=6), 50, 6),
    ("tsvd", dict(n_components=2, algorithm="bogus"), 50, 6),
]


def main():
    ref, pca, tsvd = install()
    da = ref.da
    manifest = {"reference": "mrocklin/dask-ml @ 0310a90 decomposition/pca.py, truncated_svd.py run through "
                             "tests/golden/ref_decomposition.py", "cases": {}, "errors": []}
    for name, (kind, n, d, seed, off, dt, chunks, kw) in CASES.items():
        X = data(n, d, seed, off, dt)
        Xd = da.from_array(X, chunks=(chunks, d))
        est = (pca.PCA if kind == "pca" else tsvd.TruncatedSVD)(**kw)
        T = np.asarray(est.fit_transform(Xd).compute())
        est2 = (pca.PCA if kind == "pca" else tsvd.TruncatedSVD)(**kw).fit(da.from_array(X, chunks=(chunks, d)))
        Xt = da.from_array(X[:300], chunks=(150, d))
        out = dict(X=X, chunks=chunks, fit_transform=T, transform=np.asarray(est2.transform(Xt).compute()),
                   components=np.asarray(est.components_), explained_variance=np.asarray(est.explained_variance_),
                   explained_variance_ratio=np.asarray(est.explained_variance_ratio_),
                   singular_values=np.asarray(est.singular_values_),
                   fit_components=np.asarray(est2.components_))
        Tt = da.from_array(np.asarray(out["transform"]), chunks=(150, out["transform"].shape[1]))
        out["inverse_transform"] = np.asarray(est2.inverse_transform(Tt).compute())
        if kind == "pca":
            out["mean"] = np.asarray(est.mean_.compute() if hasattr(est.mean_, "compute") else est.mean_)
            out["noise_variance"] = np.asarray(est.noise_variance_)
            out["n_components_"] = int(est.n_components_)
            out["score_samples"] = np.asarray(est2.score_samples(Xt).compute())
            out["score"] = np.asarray(est2.score(Xt).compute())
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
        manifest["cases"][name] = dict(estimator=kind, n=n, d=d, seed=seed, offset=off, dtype=dt, chunks=chunks,
                                       params=kw, singular_values=[float(v) for v in out["singular_values"]])
        print(name, manifest["cases"][name], flush=True)
    for kind, kw, n, d in ERRORS:
        X = data(n, d, 9, 0.0, "float64")
        try:
            (pca.PCA if kind == "pca" else tsvd.TruncatedSVD)(**kw).fit(da.from_array(X, chunks=(max(1, n // 2), d)))
            rec = dict(estimator=kind, params=kw, n=n, d=d, error=None, message=None)
        except Exception as e:                             # the reference's own exception type and message
            rec = dict(estimator=kind, params=kw, n=n, d=d, error=type(e).__name__, message=str(e))
        manifest["errors"].append(rec)
        print(rec, flush=True)
    with open(os.path.join(HERE, "REF_DECOMPOSITION_MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1)


if __name__ == "__main__":
    main()
