"""TEST INFRASTRUCTURE — run the UNMODIFIED reference ``LabelEncoder`` and ``OneHotEncoder``
(dask_ml/preprocessing/label.py, _encoders.py) without dask.

    BKM_REFERENCE=<dask-ml checkout> python tests/golden/ref_encoders.py   # regenerates tests/golden/ref_enc_*.npz

Built on ``ref_shim.install()``.  The encoders need a few more pieces, added here:
  * ``dask.is_dask_collection`` and ``da.unique(..., return_inverse=)`` (numpy's unique of the whole array, the inverse
    in the input's row chunks);
  * ``map_blocks`` (the method and ``da.map_blocks``) that keeps the blocks a function returns, scipy.sparse matrices
    included, and checks them against the ``new_axis`` / ``chunks`` it is given; ``da.concatenate(..., axis=1)``
    stacking the blocks of each row chunk side by side;
  * ``sklearn.preprocessing.label`` as an alias of ``sklearn.preprocessing._label``;
  * while _encoders.py is executed, a stand-in base class in place of scikit-learn's ``OneHotEncoder``: scikit-learn
    1.9's constructor is keyword-only (the reference passes its six arguments positionally) and its ``transform`` no
    longer calls ``_transform_new``.  The stand-in maps the positional arguments to scikit-learn's names
    (``sparse`` -> ``sparse_output``; ``n_values`` and ``categorical_features`` are kept as attributes only) and routes
    ``transform`` of dask-like input to ``_transform_new``; numpy input goes to scikit-learn's own ``fit`` /
    ``transform``, as in the reference.
The reference files are loaded with importlib, byte for byte.  Cases: LabelEncoder on chunked int64, float64 with NaN
and bool (fit, fit_transform, transform, inverse_transform), its unseen-label error, its numpy branch and a pandas
categorical Series; OneHotEncoder on 3-column int data (sparse and dense, float32 ``dtype``), user categories, a NaN
column and every error of the reference.  Behaviour this package does not share carries ``expected_difference``.
tests/test_encoders_host.py and tests/test_gpu_encoders.py replay the fixtures; neither needs the reference checkout.
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np
import scipy.sparse

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import ref_shim  # noqa: E402


class Blocks(ref_shim.Array):
    """A row-chunked stand-in array whose blocks are kept as returned (numpy or scipy.sparse)."""

    def __init__(self, blocks):
        self.blocks = list(blocks)

    @property
    def shape(self):
        return (sum(b.shape[0] for b in self.blocks),) + tuple(self.blocks[0].shape[1:])

    @property
    def chunks(self):
        return (tuple(b.shape[0] for b in self.blocks),) + tuple((s,) for s in self.blocks[0].shape[1:])

    def compute(self):
        if scipy.sparse.issparse(self.blocks[0]):
            return scipy.sparse.vstack(self.blocks, format="csr")
        return np.concatenate([np.asarray(b) for b in self.blocks], axis=0)


def _map(func, arrays_and_args, kwargs):
    """Apply func block by block; the stand-in arrays among the arguments supply their i-th block."""
    new_axis = kwargs.pop("new_axis", None)
    chunks = kwargs.pop("chunks", None)
    for k in ("dtype", "drop_axis"):
        kwargs.pop(k, None)
    src = next(a for a in arrays_and_args if isinstance(a, ref_shim.Array))
    out = []
    for i in range(len(src.blocks)):
        call = [a.blocks[i] if isinstance(a, ref_shim.Array) else a for a in arrays_and_args]
        out.append(func(*call, **kwargs))
    if chunks is not None:                      # what dask would be told the blocks are
        rows = chunks[0]
        assert tuple(b.shape[0] for b in out) == tuple(rows), (rows, [b.shape for b in out])
        if new_axis is not None:
            assert all(b.shape[1:] == tuple(c[0] if isinstance(c, tuple) else c for c in chunks[1:]) for b in out)
    return Blocks(out)


def install():
    ref = ref_shim.install()
    da, Array = ref.da, ref.da.Array
    dask = sys.modules["dask"]
    dask.is_dask_collection = lambda x: isinstance(x, Array)
    Array.map_blocks = lambda self, func, *args, **kwargs: _map(func, [self, *args], kwargs)
    da.map_blocks = lambda func, *args, **kwargs: _map(func, list(args), kwargs)

    def unique(values, return_inverse=False):
        full = values.compute()
        if return_inverse:
            u, inv = np.unique(full, return_inverse=True)
            return Array([u]), values._like(inv.reshape(-1))
        return Array([np.unique(full)])

    da.unique = unique
    shim_concat = da.concatenate

    def concatenate(arrs, axis=0):
        if axis != 1:
            return shim_concat(arrs, axis)
        parts = list(zip(*[a.blocks for a in arrs]))
        hs = [scipy.sparse.hstack(p, format="csr") if scipy.sparse.issparse(p[0]) else np.hstack(p) for p in parts]
        return Blocks(hs)

    da.concatenate = concatenate

    import sklearn.preprocessing
    import sklearn.preprocessing._label as sklabel

    sys.modules["sklearn.preprocessing.label"] = sklabel
    sklearn.preprocessing.label = sklabel

    root = os.path.join(ref_shim.REF, "dask_ml")
    pkg = types.ModuleType("dask_ml.preprocessing")
    pkg.__path__ = [os.path.join(root, "preprocessing")]
    sys.modules["dask_ml.preprocessing"] = pkg

    def load(name, fname):
        spec = importlib.util.spec_from_file_location(name, os.path.join(root, "preprocessing", fname))
        m = importlib.util.module_from_spec(spec)
        sys.modules[name] = m
        spec.loader.exec_module(m)
        return m

    label = load("dask_ml.preprocessing.label", "label.py")
    SkOHE = sklearn.preprocessing.OneHotEncoder

    class OneHotBase(SkOHE):
        def __init__(self, n_values=None, categorical_features=None, categories="auto", sparse=True,
                     dtype=np.float64, handle_unknown="error"):
            SkOHE.__init__(self, categories=categories, sparse_output=sparse, dtype=dtype,
                           handle_unknown=handle_unknown)
            self.n_values = n_values
            self.categorical_features = categorical_features
            self.sparse = sparse

        def transform(self, X):
            if dask.is_dask_collection(X):
                return self._transform_new(X)
            return SkOHE.transform(self, X)

    sklearn.preprocessing.OneHotEncoder = OneHotBase
    try:
        enc = load("dask_ml.preprocessing._encoders", "_encoders.py")
    finally:
        sklearn.preprocessing.OneHotEncoder = SkOHE
    return ref, label, enc


def _catch(fn):
    try:
        fn()
    except Exception as e:
        return dict(type=type(e).__name__, message=str(e))
    return None


def _csr(prefix, m):
    m = m.tocsr()
    return {prefix + "indptr": m.indptr, prefix + "indices": m.indices, prefix + "data": m.data,
            prefix + "shape": np.array(m.shape)}


def int_X(seed, n=300):
    rng = np.random.RandomState(seed)
    return np.stack([rng.randint(0, 4, n), rng.randint(-20, 20, n), rng.choice([7, -3, 1000], n)], axis=1)


def main():
    from sklearn.preprocessing import OneHotEncoder as sklearn_ohe

    ref, label, enc = install()
    da = ref.da
    manifest = {"reference": "mrocklin/dask-ml @ 0310a90 preprocessing/label.py and _encoders.py run through "
                             "tests/golden/ref_encoders.py", "label": {}, "onehot": {}, "errors": {}}
    rng = np.random.RandomState(0)

    # ---- LabelEncoder on chunked arrays ----
    ys = {"ref_enc_le_int64": rng.randint(-5, 40, 500).astype(np.int64),
          "ref_enc_le_float_nan": np.where(rng.uniform(size=500) < 0.1, np.nan, np.round(rng.standard_normal(500), 1)),
          "ref_enc_le_bool": rng.uniform(size=500) < 0.3}
    for name, y in ys.items():
        rows = 120
        le = label.LabelEncoder().fit(da.from_array(y, chunks=rows))
        out = dict(y=y, chunks=rows, classes_=np.asarray(le.classes_))
        le2 = label.LabelEncoder()
        out["fit_transform"] = np.asarray(le2.fit_transform(da.from_array(y, chunks=rows)).compute())
        entry = dict(classes_dtype=str(np.asarray(le.classes_).dtype))
        try:
            codes = np.asarray(le.transform(da.from_array(y, chunks=rows)).compute())
            out["transform"] = codes
            out["inverse"] = np.asarray(le.inverse_transform(da.from_array(codes, chunks=rows)).compute())
        except ValueError as e:
            entry["transform_error"] = str(e)
            entry["expected_difference"] = ("the reference's per-block np.setdiff1d treats NaN as unseen although "
                                             "fit made it a class; dask_ml_b200 encodes NaN as its class")
            out["inverse"] = np.asarray(le.inverse_transform(da.from_array(out["fit_transform"], chunks=rows)).compute())
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
        manifest["label"][name] = entry
        print(name, entry, flush=True)

    le = label.LabelEncoder().fit(da.from_array(ys["ref_enc_le_int64"], chunks=120))
    manifest["errors"]["le_unseen_array"] = dict(
        _catch(lambda: le.transform(da.from_array(np.array([1, 99, 3, 77]), chunks=2)).compute()),
        y=[1, 99, 3, 77], fit="ref_enc_le_int64")

    # the numpy branch: scikit-learn's fit, then np.searchsorted maps unseen labels silently
    y = np.array([3, 1, 3, 7, 1])
    le = label.LabelEncoder().fit(y)
    manifest["label"]["numpy_branch"] = dict(
        y=y.tolist(), classes_=np.asarray(le.classes_).tolist(), transform=np.asarray(le.transform(y)).tolist(),
        unseen_y=[1, 5, 100], unseen_transform=np.asarray(le.transform(np.array([1, 5, 100]))).tolist(),
        expected_difference="dask_ml_b200 raises 'previously unseen values' for unseen labels on every path")

    import pandas as pd

    s = pd.Series(pd.Categorical(["b", "a", "c", "b"], categories=["c", "b", "a"]))
    codes = label.LabelEncoder().fit_transform(s)       # (it stores the codes' dtype as dtype_: transform with a fit)
    le = label.LabelEncoder().fit(s)
    manifest["label"]["categorical"] = dict(
        values=list(s.astype(str)), categories=["c", "b", "a"], classes_=list(np.asarray(le.classes_)),
        fit_transform=np.asarray(codes).tolist(), transform=np.asarray(le.transform(s)).tolist(),
        inverse=list(le.inverse_transform(np.array([2, 0, 1])).astype(str)))

    # ---- OneHotEncoder on chunked arrays ----
    X = int_X(1)
    cases = {"ref_enc_ohe_sparse_f32": dict(sparse=True, dtype=np.float32),
             "ref_enc_ohe_dense_f32": dict(sparse=False, dtype=np.float32),
             "ref_enc_ohe_categories": dict(categories=[np.arange(6), np.arange(-20, 25), np.array([-3, 7, 1000])])}
    for name, params in cases.items():
        rows = 70
        e = enc.OneHotEncoder(**params).fit(da.from_array(X, chunks=(rows, 3)))
        t = e.transform(da.from_array(X, chunks=(rows, 3))).compute()
        out = dict(X=X, chunks=rows)
        for j, c in enumerate(e.categories_):
            out["cat%d" % j] = np.asarray(c)
        if scipy.sparse.issparse(t):
            out.update(_csr("t_", t))
        else:
            out["t"] = np.asarray(t)
        entry = dict(params={k: (v if k != "categories" else [np.asarray(c).tolist() for c in v]) if k != "dtype"
                             else np.dtype(v).name for k, v in params.items()},
                     dtypes_=[None if d is None else str(d) for d in e.dtypes_], transform_dtype=str(t.dtype))
        if np.dtype(params.get("dtype", np.float64)) != t.dtype:
            entry["expected_difference"] = ("the reference's per-block csr_matrix has float64 ones whatever `dtype` "
                                            "is; dask_ml_b200 writes `dtype`")
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
        manifest["onehot"][name] = entry
        print(name, entry, flush=True)

    Xn = np.stack([np.round(rng.uniform(size=200) * 3), rng.randint(0, 3, 200).astype(np.float64)], axis=1)
    Xn[::9, 0] = np.nan
    e = enc.OneHotEncoder(sparse=False).fit(da.from_array(Xn, chunks=(50, 2)))
    np.savez_compressed(os.path.join(HERE, "ref_enc_ohe_nan.npz"), X=Xn, chunks=50,
                        **{"cat%d" % j: np.asarray(c) for j, c in enumerate(e.categories_)})
    manifest["onehot"]["ref_enc_ohe_nan"] = dict(
        params=dict(sparse=False), transform_error=_catch(lambda: e.transform(da.from_array(Xn, chunks=(50, 2)))),
        expected_difference="the reference's np.setdiff1d rejects NaN at transform although fit made it a category; "
                            "dask_ml_b200 encodes it")

    # ---- errors ----
    arr = da.from_array(X, chunks=(70, 3))
    errs = {
        "handle_unknown_ignore": (dict(handle_unknown="ignore"), arr),
        "handle_unknown_other": (dict(handle_unknown="foo"), arr),
        "unsorted_categories": (dict(categories=[[3, 1, 2], [0], [0]]), arr),
        "shape_mismatch": (dict(categories=[[0, 1, 2, 3]]), arr),
        "unknown_at_fit_numpy": (dict(categories=[np.arange(4), np.arange(-10, 20), np.array([-3, 7, 1000])]), X),
    }
    for key, (params, src) in errs.items():
        manifest["errors"][key] = dict(
            _catch(lambda: enc.OneHotEncoder(**params).fit(src)),
            params={k: [np.asarray(c).tolist() for c in v] if k == "categories" else v for k, v in params.items()},
            input="array" if src is arr else "numpy")
    sk = _catch(lambda: sklearn_ohe(categories=errs["unknown_at_fit_numpy"][0]["categories"]).fit(X))
    manifest["errors"]["unknown_at_fit_numpy"].update(
        sklearn_message=sk["message"],
        expected_difference="the reference's _fit override does not take scikit-learn 1.9's ensure_all_finite, so its "
                            "numpy path raises TypeError; dask_ml_b200 raises scikit-learn 1.9's own error")
    bad = X.copy()
    bad[5, 2] = 55
    e = enc.OneHotEncoder().fit(arr)
    manifest["errors"]["unknown_at_transform"] = dict(
        _catch(lambda: e.transform(da.from_array(bad, chunks=(70, 3))).compute()), params={}, input="array",
        bad=[5, 2, 55], expected_difference="the reference's per-block message is 'Block contains previously unseen "
                                            "values'; dask_ml_b200 raises scikit-learn's 'Found unknown categories "
                                            "[...] in column j during transform'")
    with open(os.path.join(HERE, "REF_ENCODERS_MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1)


if __name__ == "__main__":
    main()
