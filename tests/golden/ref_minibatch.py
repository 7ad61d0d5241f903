"""TEST INFRASTRUCTURE — run the UNMODIFIED reference ``dask_ml/cluster/minibatch.py`` without dask.

    BKM_REFERENCE=<dask-ml checkout> python tests/golden/ref_minibatch.py   # regenerates tests/golden/ref_minibatch_*.npz

``ref_shim.install()`` provides the eager stand-in for dask.array; the block-wise fit of ``dask_ml/_partial.py`` needs a
few more names, added here: ``dask.delayed.Delayed`` (a dict-graph executor with ``.compute()``), ``dask.base.tokenize``,
``dask.sharedict.merge``, ``toolz.partial`` (``functools.partial``), ``six`` when it is absent, and ``Array.name`` /
``Array.dask`` (the graph keys of the row blocks).  The reference's ``_utils.py``, ``_partial.py`` and
``cluster/minibatch.py`` are then loaded with importlib, byte for byte.  Their ``fit`` calls the installed
scikit-learn's ``MiniBatchKMeans.partial_fit`` once per block, in the order the global numpy RNG shuffles the blocks
into; each case seeds that RNG and records the order.  tests/test_minibatch_host.py and tests/test_gpu_minibatch.py
replay the fixtures; neither needs the reference checkout.
"""
import functools
import importlib.util
import json
import os
import sys
import types
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import ref_shim  # noqa: E402


class Delayed(object):
    def __init__(self, key, dsk):
        self.key, self.dsk = key, dsk

    def compute(self):
        cache = {}

        def ev(x):
            if isinstance(x, tuple) and x and callable(x[0]):
                return x[0](*[ev(a) for a in x[1:]])
            if isinstance(x, tuple) and x in self.dsk:
                if x not in cache:
                    cache[x] = ev(self.dsk[x])
                return cache[x]
            return x

        return ev(self.key)


def _merge(*parts):
    out = {}
    for p in parts:
        out.update(p[1] if isinstance(p, tuple) else p)
    return out


def install():
    ref = ref_shim.install()
    dask = sys.modules["dask"]
    dd = types.ModuleType("dask.delayed")
    dd.Delayed = Delayed
    db = types.ModuleType("dask.base")
    db.tokenize = lambda *a, **k: "%x" % (id(a) & 0xFFFFFF)
    ds = types.ModuleType("dask.sharedict")
    ds.merge = _merge
    dask.base, dask.sharedict = db, ds            # dask.delayed stays ref_shim's function (k_means.py uses it)
    toolz = types.ModuleType("toolz")
    toolz.partial = functools.partial
    for name, mod in (("dask.delayed", dd), ("dask.base", db), ("dask.sharedict", ds), ("toolz", toolz)):
        sys.modules[name] = mod
    try:
        import six  # noqa: F401
    except ImportError:
        six = types.ModuleType("six")

        def add_metaclass(mc):
            def wrap(cls):
                body = dict(cls.__dict__)
                body.pop("__dict__", None)
                body.pop("__weakref__", None)
                return mc(cls.__name__, cls.__bases__, body)
            return wrap
        six.add_metaclass = add_metaclass
        sys.modules["six"] = six

    Array = ref.da.Array
    Array.name = property(lambda self: "x-%x" % id(self))
    Array.dask = property(lambda self: {(self.name, i, 0): b for i, b in enumerate(self.blocks)})

    def load(name, path):
        spec = importlib.util.spec_from_file_location(name, path)
        m = importlib.util.module_from_spec(spec)
        sys.modules[name] = m
        spec.loader.exec_module(m)
        return m

    root = os.path.join(ref_shim.REF, "dask_ml")
    load("dask_ml._utils", os.path.join(root, "_utils.py"))
    load("dask_ml._partial", os.path.join(root, "_partial.py"))
    return ref, load("dask_ml.cluster.minibatch", os.path.join(root, "cluster", "minibatch.py"))


def _blobs(n, d, centres, seed, dtype, std=1.0, weights=None):
    rng = np.random.RandomState(seed)
    k = len(centres)
    lab = rng.choice(k, size=n, p=weights)
    return (centres[lab] + std * rng.standard_normal((n, d))).astype(dtype)


def cases():
    """name -> (X, block rows, constructor keywords, number of fits)."""
    r = np.random.RandomState(40)
    c5 = r.uniform(-10, 10, size=(4, 5))
    c6 = r.uniform(-10, 10, size=(5, 6))
    c3 = r.uniform(-10, 10, size=(3, 3))
    tiny = np.vstack([r.uniform(-10, 10, size=(3, 4)), [[30.0, 30.0, 30.0, 30.0]]])
    X64 = _blobs(4000, 5, c5, 1, np.float64)
    return {
        "ref_minibatch_f64_blocks": (X64, 1000, dict(n_clusters=4, random_state=0), 1),
        "ref_minibatch_f32": (_blobs(5000, 6, c6, 2, np.float32), 1250, dict(n_clusters=5, random_state=1), 1),
        "ref_minibatch_random_init": (_blobs(3000, 3, c3, 3, np.float64), 600,
                                      dict(n_clusters=3, init="random", random_state=2), 1),
        "ref_minibatch_array_init": (X64, 800, dict(n_clusters=4, init=X64[:4].copy(), random_state=3), 1),
        "ref_minibatch_reassign": (_blobs(2400, 4, tiny, 4, np.float64, weights=[0.33, 0.33, 0.33, 0.01]), 200,
                                   dict(n_clusters=24, batch_size=100, reassignment_ratio=0.2, random_state=4), 1),
        "ref_minibatch_no_labels": (X64, 1000, dict(n_clusters=4, compute_labels=False, random_state=5), 1),
        "ref_minibatch_two_fits": (X64, 1000, dict(n_clusters=4, random_state=6), 2),
    }


def main():
    ref, mb = install()
    manifest = {}
    for ci, (name, (X, rows, kw, n_fits)) in enumerate(cases().items()):
        seed = 100 + ci
        nb = (len(X) + rows - 1) // rows
        np.random.seed(seed)
        orders = []
        for _ in range(n_fits):                         # the shuffles the reference's fit draws, replayed
            o = list(range(nb))
            np.random.shuffle(o)
            orders.append(o)
        np.random.seed(seed)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", FutureWarning)
            est = mb.PartialMiniBatchKMeans(**kw)
        Xd = ref.da.from_array(X, chunks=(rows, X.shape[1]))
        for _ in range(n_fits):
            est.fit(Xd)
        has_labels = hasattr(est, "labels_")
        init = kw.get("init", "k-means++")
        params = {k: v for k, v in kw.items() if k != "init"}
        np.savez_compressed(
            os.path.join(HERE, name + ".npz"), X=X, rows=rows, seed=seed, n_fits=n_fits, order=np.array(orders),
            init=init if isinstance(init, str) else np.asarray(init), params=json.dumps(params),
            centers=est.cluster_centers_, counts=est._counts, n_steps=est.n_steps_,
            labels=np.asarray(est.labels_) if has_labels else np.zeros(0, np.int32),
            inertia=np.float64(est.inertia_) if has_labels else np.nan)
        manifest[name] = dict(n=int(X.shape[0]), d=int(X.shape[1]), dtype=str(X.dtype), block_rows=rows, seed=seed,
                              params=params, init=init if isinstance(init, str) else "ndarray", order=orders,
                              n_steps=int(est.n_steps_), counts=np.asarray(est._counts, dtype=np.float64).tolist(),
                              inertia=float(est.inertia_) if has_labels else None)
        print(name, manifest[name], flush=True)
    with open(os.path.join(HERE, "REF_MINIBATCH_MANIFEST.json"), "w") as f:
        import sklearn

        json.dump({"reference": "mrocklin/dask-ml @ 0310a90 _partial.py + cluster/minibatch.py run through "
                                "tests/golden/ref_minibatch.py with scikit-learn %s" % sklearn.__version__,
                   "cases": manifest}, f, indent=1)


if __name__ == "__main__":
    main()
