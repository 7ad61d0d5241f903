"""TEST INFRASTRUCTURE — run the UNMODIFIED reference ``dask_ml/datasets.py`` without dask.

    BKM_REFERENCE=<dask-ml checkout> python tests/golden/ref_datasets.py   # regenerates tests/golden/ref_datasets_*.npz

``ref_shim.install()`` provides the eager stand-in for the slice of dask the KMeans path uses; the generators need a few
more pieces of it, added here: ``da.core.normalize_chunks`` (block sizes, block shapes and explicit sizes),
``da.random.random_state_data``, the ``normal`` / ``random`` / ``poisson`` draws of ``da.random.RandomState``,
``da.exp`` and ``Array.dot`` / ``squeeze`` / ``__neg__`` / ``__rtruediv__``.  The reference's file is then loaded with
importlib, byte for byte.

dask's per-block streams are not reproduced by the stand-in, so only what does not depend on them is recorded: output
shapes and dtypes, the exceptions (type and message) and make_regression's ``coef`` together with the Philox key seed
words the reference draws after it.  tests/test_datasets_host.py replays the fixtures without the reference checkout.
"""
import importlib.util
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import ref_shim  # noqa: E402


def _normalize_chunks(chunks, shape):
    """dask's normalize_chunks for a 2-D shape and the forms the generators document (dask refuses chunks=None, so the
    cases below always pass chunks)."""
    if isinstance(chunks, int):
        chunks = (chunks,) * len(shape)
    out = []
    for c, n in zip(chunks, shape):
        if isinstance(c, (tuple, list)):
            out.append(tuple(int(v) for v in c))
            continue
        c = n if c in (None, -1) else int(c)
        out.append(tuple([c] * (n // c) + ([n % c] if n % c else [])) or (n,))
    return tuple(out)


def install():
    ref = ref_shim.install()
    da, Array = ref.da, ref.da.Array
    Array.__array_ufunc__ = None

    def full(x):
        return x.compute() if isinstance(x, Array) else np.asarray(x)

    def rows(full_, chunks):
        rc = chunks[0] if isinstance(chunks, tuple) and chunks and isinstance(chunks[0], (tuple, list, int)) else chunks
        if isinstance(rc, int):
            rc = _normalize_chunks((rc,), (len(full_),))[0]
        out, s = [], 0
        for m in rc:
            out.append(full_[s:s + m])
            s += m
        return Array(out)

    Array.dot = lambda self, o: self._like(np.dot(self.compute(), full(o)))
    Array.squeeze = lambda self: self._like(np.squeeze(self.compute()))
    Array.__neg__ = lambda self: self._like(-self.compute())
    Array.__rtruediv__ = lambda self, o: self._bin(o, lambda a, b: b / a)
    da.exp = ref_shim._elementwise(np.exp)
    da.core.normalize_chunks = _normalize_chunks

    drawn = []

    def random_state_data(n, random_state=None):
        rs = random_state if isinstance(random_state, np.random.RandomState) else np.random.RandomState(random_state)
        words = np.frombuffer(rs.bytes(624 * n * 4), dtype="<u4").reshape(n, 624)
        drawn.append(words.copy())
        return list(words)

    RS = da.random.RandomState
    RS.normal = lambda self, loc=0.0, scale=1.0, size=None, chunks=None: rows(
        self._rs.normal(loc, scale, size=size), chunks)
    RS.random = lambda self, size=None, chunks=None: rows(self._rs.random_sample(size=size), chunks)
    RS.poisson = lambda self, lam=1.0, size=None, chunks=None: (
        lam._like(self._rs.poisson(full(lam))) if isinstance(lam, Array) else Array([self._rs.poisson(lam, size)]))
    da.random.random_state_data = random_state_data

    sys.modules["dask_ml"].utils = ref.utils                      # `import dask_ml.utils` binds the attribute
    spec = importlib.util.spec_from_file_location("dask_ml.datasets", os.path.join(ref_shim.REF, "dask_ml", "datasets.py"))
    ds = importlib.util.module_from_spec(spec)
    sys.modules["dask_ml.datasets"] = ds
    spec.loader.exec_module(ds)
    return ds, drawn


SHAPE_CASES = {
    # name: (function, keywords)
    "counts_default": ("make_counts", dict(random_state=0)),
    "counts_300x7": ("make_counts", dict(n_samples=300, n_features=7, n_informative=3, chunks=64, random_state=1)),
    "clf_default": ("make_classification", dict(chunks=50, random_state=0)),
    "clf_500x12": ("make_classification", dict(n_samples=500, n_features=12, n_informative=5, chunks=(128, 12),
                                               random_state=2)),
    "reg_default": ("make_regression", dict(chunks=100, random_state=0)),
    "reg_targets": ("make_regression", dict(n_samples=400, n_features=6, n_targets=3, chunks=150, noise=0.5,
                                            random_state=3)),
    "reg_one_feature_chunk": ("make_regression", dict(n_samples=200, n_features=5, chunks=((120, 80), (5,)),
                                                      random_state=4)),
}

ERROR_CASES = {
    "clf_int_chunks_below_d": ("make_classification", dict(n_samples=100, n_features=20, chunks=10)),
    "clf_column_block": ("make_classification", dict(n_samples=100, n_features=20, chunks=(50, 5))),
    "clf_explicit_columns": ("make_classification", dict(n_samples=100, n_features=4, chunks=((50, 50), (2, 2)))),
    "clf_n_classes_3": ("make_classification", dict(n_samples=100, n_features=4, n_classes=3, chunks=50)),
    "reg_column_block": ("make_regression", dict(n_samples=100, n_features=10, chunks=(20, 3))),
    "reg_int_chunks_below_d": ("make_regression", dict(n_samples=100, n_features=30, chunks=25)),
}

COEF_CASES = {
    "coef_default": dict(n_samples=100, n_features=100, chunks=100, random_state=0),
    "coef_chunks_50": dict(n_samples=1000, n_features=20, n_informative=5, chunks=50, random_state=7),
    "coef_chunks_333": dict(n_samples=1000, n_features=20, n_informative=5, chunks=333, random_state=7),
    "coef_explicit": dict(n_samples=1000, n_features=20, n_informative=5, chunks=((600, 400), (20,)), random_state=7),
    "coef_targets_3": dict(n_samples=500, n_features=8, n_informative=4, n_targets=3, chunks=100, random_state=11),
    "coef_no_shuffle": dict(n_samples=500, n_features=8, n_informative=4, shuffle=False, chunks=100, random_state=11),
    "coef_low_rank": dict(n_samples=500, n_features=15, n_informative=6, effective_rank=3, tail_strength=0.2,
                          chunks=200, random_state=12),
    "coef_bias_noise": dict(n_samples=300, n_features=10, n_informative=10, bias=2.5, noise=3.0, chunks=100,
                            random_state=13),
}


def main():
    ds, drawn = install()
    manifest = {"shapes": {}, "errors": {}, "coef": {}}
    for name, (fn, kw) in SHAPE_CASES.items():
        out = getattr(ds, fn)(**kw)
        X, y = out[0], out[1]
        manifest["shapes"][name] = dict(function=fn, kwargs=kw, X_shape=list(X.shape), X_dtype=str(X.dtype),
                                        y_shape=list(y.shape), y_dtype=str(y.dtype))
    for name, (fn, kw) in ERROR_CASES.items():
        try:
            getattr(ds, fn)(**kw)
            raise AssertionError("%s did not raise" % name)
        except (ValueError, NotImplementedError) as e:
            manifest["errors"][name] = dict(function=fn, kwargs=kw, type=type(e).__name__, message=str(e))
    for name, kw in COEF_CASES.items():
        del drawn[:]
        X, y, coef = ds.make_regression(coef=True, **kw)
        np.savez_compressed(os.path.join(HERE, "ref_datasets_%s.npz" % name), coef=np.asarray(coef),
                            seed_words=drawn[0][0, :2], X_shape=np.array(X.shape), y_shape=np.array(y.shape))
        manifest["coef"][name] = dict(kwargs=kw, coef_shape=list(np.shape(coef)))
    for sect in manifest.values():
        for v in sect.values():
            v["kwargs"] = json.loads(json.dumps(v["kwargs"], default=list))
    with open(os.path.join(HERE, "REF_DATASETS_MANIFEST.json"), "w") as f:
        json.dump({"reference": "mrocklin/dask-ml @ 0310a90 datasets.py run through tests/golden/ref_datasets.py",
                   **manifest}, f, indent=1)
    print(json.dumps(manifest, indent=1)[:3000])


if __name__ == "__main__":
    main()
