"""TEST INFRASTRUCTURE — run the UNMODIFIED reference ``dask_ml/cluster/spectral.py`` without dask.

    BKM_REFERENCE=<dask-ml checkout> python tests/golden/ref_spectral.py   # regenerates tests/golden/ref_spectral_*.npz

``ref_shim.install()`` provides the eager stand-in for the slice of dask the KMeans path uses; the spectral path needs a
few more pieces of it, added here: numpy scalars must defer to the stand-in (``__array_ufunc__ = None``), ``Array.dot``,
``Array.reshape``, ``Array.__rtruediv__``, ``da.exp``, ``da.multiply``, ``da.diag`` and a ``da.vstack`` that stacks
the rows of its arguments.  The reference's file is then loaded with importlib, byte for byte.

What each fit computed is recorded without touching the reference's code: the embedding ``U2`` through a recording
estimator passed as ``assign_labels`` (or, for the default ``'kmeans'`` branch, by replacing the module's ``KMeans``
name with a recorder, which also captures the seed the reference draws before the keep rows), and the keep rows through
a ``RandomState`` whose ``choice`` keeps its result.  tests/test_spectral_host.py and tests/test_gpu_spectral.py replay
the fixtures; neither needs the reference checkout.
"""
import importlib.util
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import ref_shim  # noqa: E402


class RecordingRandomState(np.random.RandomState):
    """A RandomState that remembers what ``choice`` returned (the reference's keep rows, before its sort)."""

    def choice(self, *a, **k):
        out = super().choice(*a, **k)
        self.chosen = np.array(out, copy=True)
        return out


def install():
    ref = ref_shim.install()
    da, Array = ref.da, ref.da.Array
    Array.__array_ufunc__ = None                                  # np.float64 * Array -> Array.__rmul__

    def full(x):
        return x.compute() if isinstance(x, Array) else np.asarray(x)

    Array.dot = lambda self, o: self._like(np.dot(self.compute(), full(o)))
    Array.reshape = lambda self, *shape: Array([self.compute().reshape(*shape)])
    Array.__rtruediv__ = lambda self, o: self._bin(o, lambda a, b: b / a)
    da.exp = ref_shim._elementwise(np.exp)
    da.multiply = lambda a, b: Array([np.multiply(full(a), full(b))])
    da.diag = lambda v: Array([np.diag(full(v))])
    da.vstack = lambda arrs: Array([np.vstack([full(a) for a in arrs])])

    spec = importlib.util.spec_from_file_location(
        "dask_ml.cluster.spectral", os.path.join(ref_shim.REF, "dask_ml", "cluster", "spectral.py"))
    sp = importlib.util.module_from_spec(spec)
    sys.modules["dask_ml.cluster.spectral"] = sp
    spec.loader.exec_module(sp)
    return ref, sp


def _recorder_class():
    from sklearn.base import BaseEstimator

    class Recorder(BaseEstimator):
        def __init__(self, n_clusters=8, random_state=None):
            self.n_clusters = n_clusters
            self.random_state = random_state

        def fit(self, X, y=None):
            self.U2_ = np.asarray(X, dtype=np.float64)
            self.labels_ = np.zeros(len(self.U2_), dtype=np.int64)
            return self

    return Recorder


def _blobs(n, d, k, seed, dtype):
    rng = np.random.RandomState(seed)
    cent = rng.uniform(-3, 3, size=(k, d))
    return (cent[rng.randint(0, k, size=n)] + 0.5 * rng.standard_normal((n, d))).astype(dtype)


def cases():
    """name -> (X, chunks, constructor keywords, branch).  branch 'kmeans' = the default label assignment."""
    from dask_ml_b200.datasets import make_blobs

    X3 = _blobs(600, 3, 3, 4, np.float32)
    X3 = ((X3 - X3.mean(0)) / X3.std(0)).astype(np.float32)
    Xb, _ = make_blobs(n_samples=200, chunks=100, random_state=0)      # the reference's test_basic data
    return {
        "ref_spectral_f64_2000x5": (_blobs(2000, 5, 4, 3, np.float64), 500,
                                    dict(n_clusters=4, n_components=40, gamma=0.2, random_state=5), "recorder"),
        "ref_spectral_f32_gamma_none": (X3, 200, dict(n_clusters=3, n_components=30, gamma=None, random_state=1),
                                        "recorder"),
        "ref_spectral_kmeans_branch": (_blobs(500, 4, 3, 8, np.float64), 250,
                                       dict(n_clusters=3, n_components=30, gamma=0.5, random_state=0), "kmeans"),
        "ref_spectral_test_basic": (np.asarray(Xb.compute(), dtype=np.float64), 100,
                                    dict(n_components=25, random_state=0), "kmeans"),
    }


def main():
    ref, sp = install()
    Recorder = _recorder_class()
    manifest = {}
    for name, (X, chunks, kw, branch) in cases().items():
        kw = dict(kw)
        seed = int(kw.pop("random_state"))
        rs = RecordingRandomState(seed)
        Xd = ref.da.from_array(X, chunks=(chunks, X.shape[1]))
        made = []
        if branch == "kmeans":
            orig = sp.KMeans

            def km(n_clusters=8, random_state=None):
                r = Recorder(n_clusters=n_clusters, random_state=random_state)
                made.append(r)
                return r

            sp.KMeans = km
            try:
                est = sp.SpectralClustering(random_state=rs, **kw).fit(Xd)
            finally:
                sp.KMeans = orig
            rec = made[0]
            km_seed = int(rec.random_state)
        else:
            rec = Recorder()
            est = sp.SpectralClustering(random_state=rs, assign_labels=rec, **kw).fit(Xd)
            km_seed = -1
        keep = np.sort(rs.chosen)
        S = np.asarray(est.eigenvalues_, dtype=np.float64)
        gamma = kw.get("gamma", 1.0)
        np.savez_compressed(os.path.join(HERE, name + ".npz"), X=X, chunks=chunks, keep=keep, U2=rec.U2_, S=S,
                            n_clusters=kw.get("n_clusters", 8), n_components=kw["n_components"],
                            gamma=np.nan if gamma is None else gamma, seed=seed, km_seed=km_seed)
        manifest[name] = dict(n=int(X.shape[0]), d=int(X.shape[1]), dtype=str(X.dtype), branch=branch,
                              n_clusters=int(kw.get("n_clusters", 8)), n_components=int(kw["n_components"]),
                              gamma=gamma, seed=seed, km_seed=km_seed, eigenvalues=S.tolist())
        print(name, manifest[name], flush=True)
    with open(os.path.join(HERE, "REF_SPECTRAL_MANIFEST.json"), "w") as f:
        json.dump({"reference": "mrocklin/dask-ml @ 0310a90 cluster/spectral.py run through tests/golden/ref_spectral.py",
                   "cases": manifest}, f, indent=1)


if __name__ == "__main__":
    main()
